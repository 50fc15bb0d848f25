"""Blockwise FP8 quantisers (b200_fp8_quantize, quantize_fp8): 1 x 128 and 128 x 128 blocks of a bf16 / fp16 / fp32
matrix, with an optional transposed copy, under the rule of the FP8-output epilogue (test_fp8_out_gpu's quant_dynamic).

The oracle is numpy on the exact fp32 values of the input: per block d = rn(amax / F) (1 when 0, NaN for a NaN / inf
block) and q = fp8(rn(x / d)).  The 1 x 128 transposed output is the 1 x 128 quantisation of x^T; the 128 x 128 one is
q^T.  Every output must equal it bit for bit, with nothing written outside the outputs.

The argument checks, the Python refusals, the oracles themselves and the build log need no GPU."""
import numpy as np
import pytest

import test_build_resources as res
from test_fp8_blockwise_gpu import MAX_INDEX, cdiv, exact_and_weight, rel_bound
from test_fp8_gpu import E4M3, E5M2, _has_gpu, decode
from test_fp8_out_gpu import FMAX, SC_SENTINEL, Case, fp8_sat, quant_dynamic, same_f32, same_fp8

try:
    import torch
except ImportError:          # the CPU argument checks need no torch
    torch = None

gpu = pytest.mark.gpu
need_torch = pytest.mark.skipif(torch is None, reason="needs torch")
IN_F32, IN_BF16, IN_F16 = 0, 1, 2                      # B200_OUT_* codes as element types
IN_NAME = {IN_F32: "f32", IN_BF16: "bf16", IN_F16: "f16"}
IN_BYTES = {IN_F32: 4, IN_BF16: 2, IN_F16: 2}
CT_NAME = {E4M3: "e4m3", E5M2: "e5m2"}
ERR_BAD_ARG, ERR_NO_DEVICE = -1, -2


def in_dtype(t):
    return {IN_F32: torch.float32, IN_BF16: torch.bfloat16, IN_F16: torch.float16}[t]


def kernel_name(in_type, ct, block, trans):
    return f"fp8_quant_{'t_' if trans else ''}{IN_NAME[in_type]}_{CT_NAME[ct]}_{'1x128' if block == 1 else '128x128'}"


# ==== the numpy oracles ============================================================================================
def quant_128x128(v, ct):
    """(bytes, d): the 128 x 128 quantisation of v (m x n float32); d is (ceil(m / 128), ceil(n / 128))."""
    m, n = v.shape
    qm, qn = cdiv(m, 128), cdiv(n, 128)
    vp = np.zeros((qm * 128, qn * 128), np.float32)
    vp[:m, :n] = v
    blocks = vp.reshape(qm, 128, qn, 128)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        bad = ~np.isfinite(blocks).all(axis=(1, 3))
        amax = np.where(np.isfinite(blocks), np.abs(blocks), 0).max(axis=(1, 3)).astype(np.float32)
        d = (amax / FMAX[ct]).astype(np.float32)
        d[d == 0] = 1
        d[bad] = np.nan
        full = np.repeat(np.repeat(d, 128, axis=0), 128, axis=1)[:m, :n]
        y = (v / full).astype(np.float32)
    return fp8_sat(y, ct), d


def oracle(v, ct, block, trans):
    """(q, s, qt, st) of one matrix; qt / st None without trans, st None for 128 x 128 (the scales are shared)."""
    if block == 1:
        q, s = quant_dynamic(v, ct)
        qt, st = quant_dynamic(np.ascontiguousarray(v.T), ct) if trans else (None, None)
    else:
        q, s = quant_128x128(v, ct)
        qt, st = (np.ascontiguousarray(q.T), None) if trans else (None, None)
    return q, s, qt, st


def test_oracles_follow_the_rule():
    """The oracles against a direct per-block loop, and the rule's corner cases: all zero (d = 1), -0 kept, NaN and inf
    blocks (d = NaN), saturation at +-F, and the transposed 1 x 128 output is the 1 x 128 quantisation of x^T."""
    rng = np.random.default_rng(1)
    for ct in (E4M3, E5M2):
        F = FMAX[ct]
        v = (rng.standard_normal((200, 300)) * np.exp2(rng.integers(-20, 20, (200, 1)))).astype(np.float32)
        v[0:128, 0:128] = 0
        v[0, 5] = -0.0
        v[130, 140] = np.nan
        v[150, 290] = -np.inf
        q, d = quant_128x128(v, ct)
        assert d.shape == (2, 3) and d[0, 0] == 1 and np.isnan(d[1, 1]) and np.isnan(d[1, 2])
        assert decode(q[0:1, 5:6], ct)[0, 0] == 0 and np.signbit(decode(q[0:1, 5:6], ct)[0, 0])
        for bi in range(2):
            for bj in range(3):
                blk = v[128 * bi:128 * bi + 128, 128 * bj:128 * bj + 128]
                if not np.isfinite(blk).all():
                    assert np.isnan(d[bi, bj]) and np.isnan(decode(q[128 * bi:128 * bi + 128, 128 * bj:128 * bj + 128], ct)).all()
                    continue
                amax = np.float32(np.abs(blk).max())
                want = np.float32(amax / F) if amax / F != 0 else np.float32(1)
                assert d[bi, bj] == want
                assert np.array_equal(q[128 * bi:128 * bi + blk.shape[0], 128 * bj:128 * bj + blk.shape[1]],
                                      fp8_sat((blk / want).astype(np.float32), ct))
        # the largest |x| of each block maps to +-F exactly (or saturates onto it); past FLT_MAX / F the scale is finite
        big = np.float32([[3.4e38, -3.4e38, 1.0]])
        qb, db = quant_dynamic(big, ct)
        assert np.isfinite(db[0, 0]) and abs(decode(qb, ct)[0, 0]) == F and decode(qb, ct)[0, 1] == -F
        qt, st = oracle(v, ct, 1, True)[2:]
        assert qt.shape == (300, 200) and st.shape == (300, 2)
        q2, s2 = quant_dynamic(np.ascontiguousarray(v.T), ct)
        assert np.array_equal(qt, q2) and same_f32(st, s2)
        qt128 = oracle(v, ct, 128, True)[2]
        assert np.array_equal(qt128, q.T)


# ==== the C ABI through ctypes =====================================================================================
def call(gemm, in_type=IN_BF16, ct=E4M3, block=1, rows=4, cols=4, batch=1, x=16, ldx=None, stride_x=0, q=16, ldq=None,
         stride_q=None, s=16, s_row=None, s_blk=1, s_entry=None, qt=None, ldqt=None, stride_qt=None, st=None,
         st_row=None, st_blk=1, st_entry=None):
    qr, qc = cdiv(rows, 128), cdiv(cols, 128)
    ldx = cols if ldx is None else ldx
    ldq = cols if ldq is None else ldq
    ldqt = rows if ldqt is None else ldqt
    stride_q = rows * ldq if stride_q is None else stride_q
    stride_qt = cols * ldqt if stride_qt is None else stride_qt
    s_row = qc if s_row is None else s_row
    s_entry = (rows if block == 1 else qr) * qc if s_entry is None else s_entry
    st_row = qr if st_row is None else st_row
    st_entry = cols * qr if st_entry is None else st_entry
    return gemm.lib.b200_fp8_quantize(in_type, ct, block, rows, cols, batch, x, ldx, stride_x, q, ldq, stride_q, s, s_row,
                                      s_blk, s_entry, qt, ldqt, stride_qt, st, st_row, st_blk, st_entry, None)


def test_argument_validation(gemm):
    """Every refusal before the device is touched, each at its bound: they hold with or without a GPU."""
    assert call(gemm, in_type=3) == ERR_BAD_ARG and call(gemm, in_type=-1) == ERR_BAD_ARG
    assert call(gemm, ct=2) == ERR_BAD_ARG and call(gemm, ct=-1) == ERR_BAD_ARG
    for block in (0, 2, 64, 127, 129, -1):
        assert call(gemm, block=block) == ERR_BAD_ARG, block
    for kw in ("rows", "cols", "batch", "stride_x", "stride_q", "s_row", "s_blk", "s_entry", "stride_qt", "st_row",
               "st_blk", "st_entry"):
        assert call(gemm, **{kw: -1}) == ERR_BAD_ARG, kw
    assert call(gemm, rows=0, ct=2) == ERR_BAD_ARG and call(gemm, batch=0, block=3) == ERR_BAD_ARG
    # no-op sizes, null pointers included
    for kw in ({"rows": 0}, {"cols": 0}, {"batch": 0}):
        assert call(gemm, x=None, q=None, s=None, ldx=0, ldq=0, **kw) == 0, kw
    # pitches below their minimum
    assert call(gemm, rows=5, cols=7, ldx=6) == ERR_BAD_ARG and call(gemm, rows=5, cols=7, ldq=6) == ERR_BAD_ARG
    assert call(gemm, rows=5, cols=7, qt=16, st=16, ldqt=4) == ERR_BAD_ARG
    # null pointers with work to do; dScaleT exactly with dQt for 1 x 128, never for 128 x 128
    for kw in ({"x": None}, {"q": None}, {"s": None}, {"qt": 16}, {"st": 16}, {"block": 128, "qt": 16, "st": 16},
               {"block": 128, "st": 16}):
        assert call(gemm, **kw) == ERR_BAD_ARG, kw
    # scale layouts that could overlap (rows = 4, cols = 300: q_c = 3), for s and st
    for sr, sb in ((2, 1), (3, 0), (1, 3), (0, 4), (3, 3), (4, 2)):
        assert call(gemm, rows=4, cols=300, s_row=sr, s_blk=sb) == ERR_BAD_ARG, (sr, sb)
        assert call(gemm, rows=300, cols=4, qt=16, st=16, st_row=sr, st_blk=sb) == ERR_BAD_ARG, (sr, sb)
    # 128 x 128 over (ceil(rows / 128), ceil(cols / 128)) = (3, 3)
    assert call(gemm, block=128, rows=300, cols=300, s_row=2, s_blk=1) == ERR_BAD_ARG
    # overlapping entries of each output, and entry strides past 2^60 / (batch - 1)
    assert call(gemm, rows=4, cols=300, batch=2, stride_q=3 * 300 + 299) == ERR_BAD_ARG
    assert call(gemm, rows=4, cols=300, batch=2, s_entry=11) == ERR_BAD_ARG
    assert call(gemm, rows=300, cols=4, batch=2, qt=16, st=16, stride_qt=3 * 300 + 299) == ERR_BAD_ARG
    assert call(gemm, rows=300, cols=4, batch=2, qt=16, st=16, st_entry=11) == ERR_BAD_ARG
    assert call(gemm, rows=4, cols=4, batch=3, stride_x=(1 << 59) + 1) == ERR_BAD_ARG
    # a last element whose byte offset does not fit a signed 64-bit integer
    assert call(gemm, rows=4, cols=300, s_row=MAX_INDEX, s_blk=1) == ERR_BAD_ARG
    assert call(gemm, rows=4, cols=300, s_row=(1 << 63) - 1, s_blk=1) == ERR_BAD_ARG        # past 64 bits as an index
    assert call(gemm, rows=300, cols=4, qt=16, st=16, st_row=(1 << 63) - 1, st_blk=1) == ERR_BAD_ARG
    assert call(gemm, in_type=IN_F32, rows=(1 << 31) - 1, cols=4, ldx=(1 << 31) - 1) == ERR_BAD_ARG


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device behaviour")
def test_accepts_at_the_bounds_without_device(gemm):
    """Legal calls at the bounds reach the device check (-2)."""
    for in_type in (IN_F32, IN_BF16, IN_F16):
        for ct in (E4M3, E5M2):
            for block in (1, 128):
                assert call(gemm, in_type=in_type, ct=ct, block=block) == ERR_NO_DEVICE
                st = 16 if block == 1 else None
                assert call(gemm, in_type=in_type, ct=ct, block=block, qt=16, st=st) == ERR_NO_DEVICE
    for sr, sb in ((3, 1), (9, 1), (1, 4), (1, 9)):                        # rows = 4, q_c = 3: both layouts, padded
        assert call(gemm, rows=4, cols=300, s_row=sr, s_blk=sb) == ERR_NO_DEVICE, (sr, sb)
        assert call(gemm, rows=300, cols=4, qt=16, st=16, st_row=sr, st_blk=sb) == ERR_NO_DEVICE, (sr, sb)
    assert call(gemm, rows=1, cols=300, s_row=0) == ERR_NO_DEVICE                # extent-1 rows: the row stride is free
    assert call(gemm, rows=4, cols=100, s_row=1, s_blk=0) == ERR_NO_DEVICE       # one block: the block stride is free
    assert call(gemm, rows=2, cols=300, s_row=MAX_INDEX - 2) == ERR_NO_DEVICE
    assert call(gemm, rows=5, cols=7, ldx=7, ldq=7, qt=16, st=16, ldqt=5) == ERR_NO_DEVICE
    assert call(gemm, rows=5, cols=7, ldx=9, ldq=11, qt=16, st=16, ldqt=13) == ERR_NO_DEVICE
    assert call(gemm, rows=4, cols=300, batch=2, stride_x=0, stride_q=4 * 300, s_entry=12) == ERR_NO_DEVICE
    assert call(gemm, rows=4, cols=4, batch=3, stride_x=1 << 59) == ERR_NO_DEVICE
    assert call(gemm, in_type=IN_F32, rows=1 << 30, cols=4, ldx=(1 << 31) - 1) == ERR_NO_DEVICE   # just inside
    assert call(gemm, block=128, rows=300, cols=300, s_row=3, s_blk=1, qt=16) == ERR_NO_DEVICE


# ==== Python: refusals (CPU) =======================================================================================
@need_torch
def test_python_refusals(gemm):
    x = torch.zeros((200, 300), dtype=torch.bfloat16)
    with pytest.raises(TypeError):
        gemm.quantize_fp8(x.to(torch.float64))
    with pytest.raises(TypeError):
        gemm.quantize_fp8(torch.zeros((4, 4), dtype=torch.int32))
    with pytest.raises(TypeError):
        gemm.quantize_fp8(x, dtype=torch.bfloat16)
    for block in ((128, 1), (1, 1), (64, 64), (1, 128, 1)):
        with pytest.raises(ValueError, match="block"):
            gemm.quantize_fp8(x, block=block)
    with pytest.raises(ValueError, match="2-D or 3-D"):
        gemm.quantize_fp8(torch.zeros(8, dtype=torch.bfloat16))
    with pytest.raises(ValueError, match="unit last stride"):
        gemm.quantize_fp8(x.t())
    with pytest.raises(ValueError, match="overlap"):
        gemm.quantize_fp8(torch.zeros(400, dtype=torch.bfloat16).as_strided((4, 300), (2, 1)))
    with pytest.raises(ValueError, match="out must"):
        gemm.quantize_fp8(x, dtype=torch.float8_e4m3fn, out=torch.empty((200, 300), dtype=torch.float8_e5m2))
    with pytest.raises(ValueError, match="out must"):
        gemm.quantize_fp8(x, out=torch.empty((300, 200), dtype=torch.float8_e4m3fn))
    with pytest.raises(ValueError, match="out_scale"):
        gemm.quantize_fp8(x, out_scale=torch.empty((2, 3)))                       # the 128 x 128 shape for 1 x 128
    with pytest.raises(ValueError, match="out_scale"):
        gemm.quantize_fp8(x, block=(128, 128), out_scale=torch.empty((200, 3)))
    with pytest.raises(ValueError, match="out_scale"):
        gemm.quantize_fp8(x, out_scale=torch.empty((200, 3), dtype=torch.float64))
    with pytest.raises(ValueError, match="out_scale"):
        gemm.quantize_fp8(x, out_scale=torch.empty(600).as_strided((200, 3), (2, 1)))
    x3 = torch.zeros((4, 200, 300), dtype=torch.float16)
    with pytest.raises(ValueError, match="entries of out must"):
        gemm.quantize_fp8(x3, out=torch.empty((200, 300), dtype=torch.float8_e4m3fn).expand(4, 200, 300))
    with pytest.raises(ValueError, match="entries of out_scale"):
        gemm.quantize_fp8(x3, out_scale=torch.empty((200, 3)).expand(4, 200, 3))
    # everything else resolves and reaches the CUDA check
    for block in ((1, 128), (128, 128)):
        for xx in (x, x3, x.float(), x[:, :299], x[:1]):
            with pytest.raises(ValueError, match="CUDA"):
                gemm.quantize_fp8(xx, block=block, transpose=True)
    for out_scale in (torch.empty((200, 3)), torch.empty((3, 200)).t()):
        with pytest.raises(ValueError, match="CUDA"):
            gemm.quantize_fp8(x, out_scale=out_scale)


def test_quantiser_kernels_do_not_spill():
    """24 kernels (3 input types x 2 FP8 types x 2 blocks x with / without the transposed output), 0 spill bytes."""
    k = res.kernels()
    names = [n for n in k if "fp8_quant_kernel" in n]
    assert len(names) == 24, names
    for n in names:
        assert k[n]["spill"] == 0, (n, k[n])


# ==== GPU ==========================================================================================================
def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def exact_values(v, in_type):
    """float32 values representable in the input type, and the device tensor of that type."""
    t = torch.from_numpy(np.ascontiguousarray(v, np.float32)).to(in_dtype(in_type))
    return t.float().numpy(), t


def random_input(rng, shape, in_type):
    """Normal values with row magnitudes spread over 2^-12 .. 2^12 (2^-6 .. 2^6 for fp16), zeros of both signs."""
    span = 6 if in_type == IN_F16 else 12
    v = rng.standard_normal(shape) * np.exp2(rng.integers(-span, span + 1, shape[:-1] + (1,)))
    v = v.astype(np.float32)
    v.reshape(-1)[::97] = 0.0
    v.reshape(-1)[1::97] = -0.0
    return v


class Buf:
    """A fenced device byte buffer: `pad` sentinel bytes on both sides of `size` bytes that start at an offset."""

    def __init__(self, size, off=0, pad=64, fill=0xA5):
        self.size, self.off, self.pad = size, off, pad
        self.t = torch.full((pad + off + size + pad,), fill, dtype=torch.uint8, device="cuda")
        self.fill = fill

    @property
    def ptr(self):
        return self.t.data_ptr() + self.pad + self.off

    def bytes(self):
        return self.t.cpu().numpy()


class SBuf:
    """A float32 scale buffer inside 8 sentinel floats on each side."""

    def __init__(self, count):
        self.count = count
        self.t = torch.full((8 + count + 8,), SC_SENTINEL, dtype=torch.int32, device="cuda")

    @property
    def ptr(self):
        return self.t.data_ptr() + 32

    def values(self):
        a = self.t.cpu().numpy()
        assert (a[:8] == SC_SENTINEL).all() and (a[8 + self.count:] == SC_SENTINEL).all()
        return a[8:8 + self.count]


def scale_strides(rows, blks, layout, pad=0):
    """(s_row, s_blk, elements of one entry) of a (rows, blks) scale matrix, row-major or outer-dim-major, with pad
    unused elements per row (or column)."""
    if layout == "row":
        return blks + pad, 1, rows * (blks + pad)
    return 1, rows + pad, blks * (rows + pad)


def run_abi(gemm, v, in_type, ct, block, trans, x_off=0, ldx_extra=0, q_off=0, ldq_extra=0, layout="row",
            entry_pad=0, stream=None):
    """b200_fp8_quantize on v ((batch, rows, cols) float32 values exact in in_type), every output fenced; returns
    [(q, s, qt, st)] per entry, checking the fences, the untouched padding, the kernel name and one launch."""
    B, m, n = v.shape
    qr, qc = cdiv(m, 128), cdiv(n, 128)
    esz = IN_BYTES[in_type]
    ldx = n + ldx_extra
    stride_x = m * ldx + entry_pad
    xv, xt = exact_values(v, in_type)
    X = torch.full((x_off + B * stride_x + 8,), float("nan"), dtype=in_dtype(in_type), device="cuda")
    X.as_strided((B, m, n), (stride_x, ldx, 1), x_off).copy_(xt.cuda())
    ldq = n + ldq_extra
    stride_q = m * ldq + entry_pad
    Q = Buf(B * stride_q, q_off)
    srows = m if block == 1 else qr
    s_row, s_blk, s_elems = scale_strides(srows, qc, layout, pad=1 if entry_pad else 0)
    s_entry = s_elems + entry_pad
    S = SBuf(B * s_entry)
    ldqt, stride_qt, st_row, st_blk, st_entry = m + ldq_extra, 0, 0, 0, 0
    QT = ST = None
    if trans:
        stride_qt = n * ldqt + entry_pad
        QT = Buf(B * stride_qt, q_off)
        if block == 1:
            st_row, st_blk, st_elems = scale_strides(n, qr, layout, pad=1 if entry_pad else 0)
            st_entry = st_elems + entry_pad
            ST = SBuf(B * st_entry)
    before = gemm.launch_count()
    rc = gemm.lib.b200_fp8_quantize(in_type, ct, block, m, n, B, X.data_ptr() + esz * x_off, ldx, stride_x, Q.ptr, ldq,
                                    stride_q, S.ptr, s_row, s_blk, s_entry, QT.ptr if QT else None, ldqt, stride_qt,
                                    ST.ptr if ST else None, st_row, st_blk, st_entry, stream)
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert gemm.launch_count() == before + 1
    assert gemm.last_kernel() == kernel_name(in_type, ct, block, trans)

    def matrices(buf, rows, cols, ld, stride):
        a = buf.bytes()
        lo, hi = buf.pad + buf.off, buf.pad + buf.off + buf.size
        assert (a[:lo] == 0xA5).all() and (a[hi:] == 0xA5).all()
        body = a[lo:hi]
        out = []
        for e in range(B):
            ent = body[e * stride:(e + 1) * stride]
            mat = ent[:rows * ld].reshape(rows, ld)
            assert (mat[:, cols:] == 0xA5).all() and (ent[rows * ld:] == 0xA5).all()    # pitch and entry padding
            out.append(np.ascontiguousarray(mat[:, :cols]))
        return out

    def scales(sb, rows, blks, sr, sk, entry):
        a = sb.values()
        out, used = [], np.zeros(a.shape, bool)
        for e in range(B):
            idx = e * entry + np.arange(rows)[:, None] * sr + np.arange(blks)[None, :] * sk
            used[idx] = True
            out.append(a[idx].view(np.float32))
        assert (a[~used] == SC_SENTINEL).all()
        return out

    qs = matrices(Q, m, n, ldq, stride_q)
    ss = scales(S, srows, qc, s_row, s_blk, s_entry)
    qts = matrices(QT, n, m, ldqt, stride_qt) if trans else [None] * B
    sts = scales(ST, n, qr, st_row, st_blk, st_entry) if ST else [None] * B
    return xv, list(zip(qs, ss, qts, sts))


def check_against_oracle(xv, got, ct, block, trans, what):
    for e, (q, s, qt, st) in enumerate(got):
        wq, ws, wqt, wst = oracle(xv[e], ct, block, trans)
        assert same_f32(s, ws), (what, e, "scales")
        assert same_fp8(q, wq, ct), (what, e, "q")
        if trans:
            assert same_fp8(qt, wqt, ct), (what, e, "qt")
            if block == 1:
                assert same_f32(st, wst), (what, e, "st")
            else:
                assert np.array_equal(qt, q.T), (what, e, "qt == q^T")


SHAPES = [(1, 129), (127, 300), (129, 1), (300, 127), (257, 384)]


@gpu
@pytest.mark.parametrize("trans", [False, True], ids=["q", "qt"])
@pytest.mark.parametrize("block", [1, 128], ids=["1x128", "128x128"])
@pytest.mark.parametrize("ct", [E4M3, E5M2], ids=lambda c: CT_NAME[c])
@pytest.mark.parametrize("in_type", [IN_BF16, IN_F16, IN_F32], ids=lambda t: IN_NAME[t])
def test_bit_exact_against_numpy(gemm, in_type, ct, block, trans):
    """Tails of 1, 127, 129 and 300 on both dimensions; aligned and unaligned bases, odd pitches, both scale layouts."""
    rng = np.random.default_rng(100 + 16 * in_type + 8 * ct + 2 * (block == 128) + trans)
    for m, n in SHAPES:
        v = random_input(rng, (1, m, n), in_type)
        for x_off, ldx_extra, q_off, ldq_extra, layout in ((0, 0, 0, 0, "row"), (1, 3, 1, 5, "outer"),
                                                           (0, 8, 3, 0, "outer"), (3, 1, 0, 16, "row")):
            xv, got = run_abi(gemm, v, in_type, ct, block, trans, x_off, ldx_extra, q_off, ldq_extra, layout)
            check_against_oracle(xv, got, ct, block, trans, (m, n, x_off, ldx_extra, q_off, ldq_extra, layout))


@gpu
@pytest.mark.parametrize("block", [1, 128], ids=["1x128", "128x128"])
@pytest.mark.parametrize("in_type", [IN_BF16, IN_F32], ids=lambda t: IN_NAME[t])
def test_batch_with_padded_entry_strides(gemm, in_type, block):
    """A batch of 5 entries, each input, output and scale entry padded apart (vector and element loads)."""
    rng = np.random.default_rng(200 + in_type + block)
    for m, n, x_off in ((130, 260, 0), (127, 129, 1)):
        v = random_input(rng, (5, m, n), in_type)
        for ct in (E4M3, E5M2):
            xv, got = run_abi(gemm, v, in_type, ct, block, True, x_off=x_off, ldx_extra=8, entry_pad=8 * 7,
                              layout="outer" if x_off else "row")
            check_against_oracle(xv, got, ct, block, True, (m, n, x_off))


@gpu
@pytest.mark.parametrize("in_type", [IN_BF16, IN_F16, IN_F32], ids=lambda t: IN_NAME[t])
def test_special_blocks(gemm, in_type):
    """All-zero blocks (d = 1), -0, a NaN, +-inf (NaN blocks), subnormals, and for fp32 values near FLT_MAX (a finite
    scale, saturation at +-F)."""
    rng = np.random.default_rng(300 + in_type)
    m, n = 300, 390
    v = random_input(rng, (m, n), in_type)
    v[0:128, 0:128] = 0.0                            # an all-zero tile: every block recipe sees d = 1
    v[3, 128:256] = -0.0                             # a 1 x 128 block of -0 only
    v[200, 5] = np.nan
    v[140, 300] = np.inf
    v[260, 150] = -np.inf
    tiny = {IN_F32: 1e-40, IN_BF16: 1e-40, IN_F16: 3e-8}[in_type]
    v[129:140, 128:256] = tiny * rng.integers(-3, 4, (11, 128))   # 1 x 128 blocks of subnormals of the input type
    if in_type == IN_F32:
        v[280, 260:300] = 3.4e38 * rng.choice([-1, 1], 40)
        v[290:299, 0] = -3.3e38
    for ct in (E4M3, E5M2):
        for block in (1, 128):
            xv, got = run_abi(gemm, v[None], in_type, ct, block, True)
            check_against_oracle(xv, got, ct, block, True, (ct, block))
            q, s, qt, st = got[0]
            if block == 1:
                assert s[0, 0] == 1 and s[3, 1] == 1 and np.isnan(s[200, 0]) and np.isnan(s[140, 2])
                assert np.signbit(decode(q[3:4, 140:141], ct)[0, 0]) and (q[3, 128:256] == 0x80).all()
                assert np.isnan(st[5, 1]) and np.isnan(st[150, 2]) and st[0, 0] == 1
            else:
                assert s[0, 0] == 1 and np.isnan(s[1, 0]) and np.isnan(s[1, 2]) and np.isnan(s[2, 1])
            if in_type == IN_F32:
                r = decode(q[280:281, 260:300], ct)
                assert np.isfinite(s[280, 2] if block == 1 else s[2, 2]) and (np.abs(r) <= FMAX[ct]).all()
                assert (np.abs(r) == FMAX[ct]).any()


@gpu
@pytest.mark.parametrize("ct", [E4M3, E5M2], ids=lambda c: CT_NAME[c])
def test_same_rule_as_the_epilogue(gemm, ct):
    """b200_gemm_fp8_blockwise's fp32 C quantised with block = 1 equals b200_gemm_fp8_blockwise_q8's (C, scale_c) on the
    same inputs, bit for bit, for both scale layouts."""
    rng = np.random.default_rng(400 + ct)
    for m, n, k in ((130, 300, 256), (77, 127, 128), (256, 384, 416)):
        case = Case(gemm, ("blk", (1, 128), 0), E4M3, E4M3, m, n, k, rng, bias=False)
        c32 = case.c32()
        for layout in ("row", "outer"):
            want_q, want_d = case.q8(ct, dynamic=True, sc_layout=layout)
            xv, got = run_abi(gemm, c32[None], IN_F32, ct, 1, False, layout=layout)
            q, s = got[0][:2]
            assert np.array_equal(q, want_q) and same_f32(s, want_d), (m, n, k, layout)


@gpu
def test_linear_layer_end_to_end(gemm):
    """A blockwise FP8 linear layer, forward, dgrad and wgrad, from quantize_fp8 and scaled_mm only: the same scaled_mm
    calls on the numpy-quantised operands give the same bits, and each product lies within the blockwise error bound
    of the float64 product of the dequantised operands."""
    torch.manual_seed(500)
    M, N, K = 384, 320, 512
    x = torch.randn((M, K), device="cuda", dtype=torch.bfloat16)
    W = (torch.randn((N, K), device="cuda") * 0.05).bfloat16()
    dy = (torch.randn((M, N), device="cuda") * 1e-3).bfloat16()
    xq, xs, xqt, xst = gemm.quantize_fp8(x, transpose=True)
    wq, ws, wqt, wst = gemm.quantize_fp8(W, block=(128, 128), transpose=True)
    dyq, dys, dyqt, dyst = gemm.quantize_fp8(dy, transpose=True)
    assert xs.shape == (M, 4) and xst.shape == (K, 3) and ws.shape == (3, 4) and wst.shape == (4, 3)
    assert wst.data_ptr() == ws.data_ptr() and wst.stride() == (1, 4)
    # the numpy quantisation of the same values
    u8 = lambda t: t.view(torch.uint8).cpu().numpy()                                       # noqa: E731
    xv, Wv, dyv = (t.float().cpu().numpy() for t in (x, W, dy))
    nx, nw, ndy = oracle(xv, E4M3, 1, True), oracle(Wv, E4M3, 128, True), oracle(dyv, E4M3, 1, True)
    for got, want in (((xq, xs, xqt, xst), nx), ((wq, ws, wqt, None), nw), ((dyq, dys, dyqt, dyst), ndy)):
        assert np.array_equal(u8(got[0]), want[0]) and same_f32(got[1].cpu().numpy(), want[1])
        assert np.array_equal(u8(got[2]), want[2])
        if got[3] is not None:
            assert same_f32(got[3].cpu().numpy(), want[3])
    f8 = lambda a: dev(a).view(torch.float8_e4m3fn)                                         # noqa: E731
    chains = {
        "forward": ((xq, wq.t(), xs, ws.t()), (f8(nx[0]), f8(nw[0]).t(), dev(nx[1]), dev(nw[1]).t())),
        "dgrad": ((dyq, wqt.t(), dys, ws), (f8(ndy[0]), f8(nw[2]).t(), dev(ndy[1]), dev(nw[1]))),
        "wgrad": ((dyqt, xqt.t(), dyst, xst.t()), (f8(ndy[2]), f8(nx[2]).t(), dev(ndy[3]), dev(nx[3]).t())),
    }
    for name, (lib_args, np_args) in chains.items():
        got = gemm.scaled_mm(*lib_args, out_dtype=torch.float32)
        want = gemm.scaled_mm(*np_args, out_dtype=torch.float32)
        assert same_f32(got.cpu().numpy(), want.cpu().numpy()), name
        A, B, sa, sb = lib_args
        a = decode(u8(A.contiguous()), E4M3)
        b = decode(u8(B.t().contiguous()), E4M3).T
        kk = a.shape[1]
        sa_full = sa.cpu().numpy()                                                          # (m, q): 1 x 128
        sb_np = sb.cpu().numpy()
        sb_full = sb_np if sb_np.shape[1] == b.shape[1] else np.repeat(sb_np, 128, axis=1)[:, :b.shape[1]]
        ex, w = exact_and_weight(a, b, sa_full, sb_full)
        err = np.abs(got.double().cpu().numpy() - ex)
        assert bool((err <= rel_bound(kk) * w).all()), (name, float((err / np.maximum(w, 1e-300)).max()))


@gpu
def test_moe_forward_and_dgrad_end_to_end(gemm):
    """An FP8 mixture-of-experts layer through scaled_grouped_mm: the forward with 1 x 128 tokens and 128 x 128 expert
    weights, and the dgrad with the weights' transposed copy, equal the same calls on numpy-quantised operands bit for
    bit and lie within the blockwise error bound."""
    torch.manual_seed(600)
    G, d, dff = 4, 384, 256
    sizes = [100, 0, 300, 57]
    T = sum(sizes)
    offs = torch.tensor(np.cumsum(sizes), dtype=torch.int32, device="cuda")
    x = torch.randn((T, d), device="cuda", dtype=torch.bfloat16)
    W = (torch.randn((G, dff, d), device="cuda") * 0.05).bfloat16()
    dy = (torch.randn((T, dff), device="cuda") * 1e-2).bfloat16()
    xq, xs = gemm.quantize_fp8(x)
    wq, ws, wqt, wst = gemm.quantize_fp8(W, block=(128, 128), transpose=True)
    assert gemm.last_kernel() == "fp8_quant_t_bf16_e4m3_128x128"
    dyq, dys = gemm.quantize_fp8(dy)
    assert wqt.shape == (G, d, dff) and ws.shape == (G, 2, 3) and wst.shape == (G, 3, 2)
    u8 = lambda t: t.view(torch.uint8).cpu().numpy()                                       # noqa: E731
    xv, dyv = x.float().cpu().numpy(), dy.float().cpu().numpy()
    nx, ndy = oracle(xv, E4M3, 1, False), oracle(dyv, E4M3, 1, False)
    nw = [oracle(W[g].float().cpu().numpy(), E4M3, 128, True) for g in range(G)]
    assert np.array_equal(u8(xq), nx[0]) and same_f32(xs.cpu().numpy(), nx[1])
    assert np.array_equal(u8(dyq), ndy[0]) and same_f32(dys.cpu().numpy(), ndy[1])
    for g in range(G):
        assert np.array_equal(u8(wq[g]), nw[g][0]) and np.array_equal(u8(wqt[g]), nw[g][2])
        assert same_f32(ws[g].cpu().numpy(), nw[g][1])
    f8 = lambda a: dev(a).view(torch.float8_e4m3fn)                                         # noqa: E731
    Wn = f8(np.stack([w[0] for w in nw]))
    Wtn = f8(np.stack([w[2] for w in nw]))
    Sn = dev(np.stack([w[1] for w in nw]))
    y = gemm.scaled_grouped_mm(xq, wq.transpose(-2, -1), xs, ws.transpose(-2, -1), offs, out_dtype=torch.float32)
    y_np = gemm.scaled_grouped_mm(f8(nx[0]), Wn.transpose(-2, -1), dev(nx[1]), Sn.transpose(-2, -1), offs,
                                  out_dtype=torch.float32)
    dx = gemm.scaled_grouped_mm(dyq, wqt.transpose(-2, -1), dys, ws, offs, out_dtype=torch.float32)
    assert gemm.last_kernel() == "tc_e4m3_of32_grp_blk_128x128"
    dx_np = gemm.scaled_grouped_mm(f8(ndy[0]), Wtn.transpose(-2, -1), dev(ndy[1]), Sn, offs, out_dtype=torch.float32)
    assert same_f32(y.cpu().numpy()[:T], y_np.cpu().numpy()[:T])
    assert same_f32(dx.cpu().numpy()[:T], dx_np.cpu().numpy()[:T])
    ends = [0] + np.cumsum(sizes).tolist()
    for g in range(G):
        lo, hi = ends[g], ends[g + 1]
        if hi == lo:
            continue
        wd = decode(nw[g][0], E4M3)                                                         # (dff, d)
        sw = nw[g][1]                                                                       # (dff / 128, d / 128)
        # forward: (x_g @ W_g^T), k = d;  dgrad: (dy_g @ W_g), k = dff
        for out, a8, sa, b, sb_full, kk in (
                (y, nx[0][lo:hi], nx[1][lo:hi], wd.T, np.repeat(sw.T, 128, axis=1)[:, :dff], d),
                (dx, ndy[0][lo:hi], ndy[1][lo:hi], wd, np.repeat(sw, 128, axis=1)[:, :d], dff)):
            ex, w = exact_and_weight(decode(a8, E4M3), b, sa, sb_full)
            err = np.abs(out[lo:hi].double().cpu().numpy() - ex)
            assert bool((err <= rel_bound(kk) * w).all()), g


@gpu
def test_past_32_bit_offsets(gemm):
    """One 128 x 128 call with the transposed output over a 16385 x 131072 bf16 matrix: x's last element is past 2^31
    elements, and so are the last rows of q and qt.  Checked on sampled tiles, the last (one-row) tile row included."""
    m, n = 16385, 131072
    torch.manual_seed(700)
    x = torch.randn((m, n), device="cuda", dtype=torch.bfloat16)
    q, s, qt, st = gemm.quantize_fp8(x, block=(128, 128), transpose=True)
    torch.cuda.synchronize()
    assert gemm.last_kernel() == "fp8_quant_t_bf16_e4m3_128x128" and s.shape == (129, 1024)
    for tr, tc in ((0, 0), (64, 511), (127, 1023), (128, 0), (128, 1023), (3, 1000)):
        rs, cs = slice(128 * tr, min(128 * tr + 128, m)), slice(128 * tc, 128 * tc + 128)
        v = x[rs, cs].float().cpu().numpy()
        wq, wd = quant_128x128(v, E4M3)
        assert same_f32(s[tr:tr + 1, tc:tc + 1].cpu().numpy(), wd), (tr, tc)
        assert np.array_equal(q[rs, cs].view(torch.uint8).cpu().numpy(), wq), (tr, tc)
        assert np.array_equal(qt[cs, rs].view(torch.uint8).cpu().numpy(), wq.T), (tr, tc)
    del q, qt
    torch.cuda.empty_cache()


@gpu
def test_cuda_graph_replay_with_new_values(gemm):
    """quantize_fp8 of both recipes with the transposed output, captured in one CUDA graph and replayed with new input
    values written in place."""
    rng = np.random.default_rng(800)
    m, n = 300, 260
    x = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
    w = torch.empty((2, m, n), dtype=torch.float32, device="cuda")
    x.copy_(torch.from_numpy(random_input(rng, (m, n), IN_BF16)))
    w.copy_(torch.from_numpy(random_input(rng, (2, m, n), IN_F32)))
    outs = {}

    def calls():
        outs["x"] = gemm.quantize_fp8(x, transpose=True)
        outs["w"] = gemm.quantize_fp8(w, block=(128, 128), dtype=torch.float8_e5m2, transpose=True)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        calls()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        calls()
    u8 = lambda t: t.view(torch.uint8).cpu().numpy()                                       # noqa: E731
    for _ in range(3):
        x.copy_(torch.from_numpy(random_input(rng, (m, n), IN_BF16)))
        w.copy_(torch.from_numpy(random_input(rng, (2, m, n), IN_F32)))
        g.replay()
        torch.cuda.synchronize()
        q, sc, qt, st = outs["x"]
        wq, ws, wqt, wst = oracle(x.float().cpu().numpy(), E4M3, 1, True)
        assert np.array_equal(u8(q), wq) and same_f32(sc.cpu().numpy(), ws)
        assert np.array_equal(u8(qt), wqt) and same_f32(st.cpu().numpy(), wst)
        q, sc, qt, st = outs["w"]
        for e in range(2):
            wq, ws, wqt, _ = oracle(w[e].cpu().numpy(), E5M2, 128, True)
            assert same_fp8(u8(q[e]), wq, E5M2) and same_f32(sc[e].cpu().numpy(), ws)
            assert same_fp8(u8(qt[e]), wqt, E5M2) and same_f32(st[e].cpu().numpy(), ws.T)
