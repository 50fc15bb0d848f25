"""Every GEMM route past the CUDA grid limits and past 2^31-element offsets.

The C ABI takes m, n and k up to INT_MAX.  gridDim.y may not exceed 65535, so a launcher that sizes grid.y from a
problem dimension must cap it and its kernel must walk y with a grid stride; otherwise a valid call fails with
cudaErrorInvalidConfiguration.  Group A runs each such launch just past its threshold:

  col_absmax_kernel (F16X2 column maxima)      ceil(rows / 16) row blocks   rows = k (row-major B, A^T)
  transpose_kernel (tf32 / int8 / FP8 / STRICT) ceil(rows / 32) row tiles    rows = k (row-major B, A^T), n (B^T)
  gemm_generic_kernel and its batched form      ceil(m / 64) row blocks      every unaligned-pitch call
  mxf4_quantize_cols_t / mxf4_expand_cols_t     kpad / 32 K-blocks           b200_mxf4_quantize_b, b200_gemm_mxf4

Group B runs operands and outputs of more than 2^31 elements (or bytes), so that every offset on those paths must be
computed in 64 bits.  Each case declares its footprint and is skipped, with the free memory in the reason, when the
device has less than 1.25 times that free; nothing probes by allocating.

Operands are small integers (values in [-2, 2], int8 in [-1, 1], exact FP8 integers, power-of-two scales), chosen so
that every product and every partial sum is an integer (or a dyadic with few bits) below 2^24: exact in fp32, so every
route, whatever its accumulation order, K split or plane split, must equal the float64 product bit for bit.  Output
buffers start as NaN (int32: a sentinel) with padding columns that must stay so, operands carry NaN in their padding,
whole outputs are compared in row chunks, and last_kernel() names the route each case must take.

The case table and the exactness bounds are checked without a GPU."""
import numpy as np
import pytest

import _libs
from test_transposed_ops_gpu import hooks  # noqa: F401  (fixture: scheduling hooks reset)

try:
    import torch
except ImportError:          # the CPU tests need no torch
    torch = None

gpu = pytest.mark.gpu
MAX_GRID_Y = 65535
EXACT = 1 << 24              # every integer below this is exact in fp32

# ==== the case table ================================================================================================
# Group A extents: each just past its threshold, not a power of two, and not a multiple of its tile (the last row block
# is partial), so the capped grid walks a partial second round.
F16X2_K = 1048576 + 104      # col_absmax_kernel: ceil(k / 16) = 65543 row blocks; a multiple of 8 (TMA pitch of fp32)
XPOSE_K = 2097152 + 176      # transpose_kernel: ceil(k / 32) = 65542 row tiles; a multiple of 16 (int8 / FP8 TMA pitch)
GENERIC_M = (1 << 22) + 77   # gemm_generic_kernel: ceil(m / 64) = 65538 row blocks
MXF4_K = (1 << 21) + 100     # kpad = 2^21 + 128: 65540 K-blocks of 32
GEN_K, GEN_N = 24, 40        # the generic cases' k and n; lda = k + 1 is no 16-byte multiple for any operand type

# (name, extent, tile of grid.y, operand magnitudes (|a|, |b|), k of the accumulation, extra magnitude added in the
# epilogue).  The CPU tests check grid.y > 65535 and max |partial sum| < 2^24 from this table.
GRID_CASES = [
    ("f16x2", F16X2_K, 16, (2, 2), F16X2_K, 0),
    ("strict_tn", XPOSE_K, 32, (2, 2), XPOSE_K, 0),
    ("strict_nt", XPOSE_K, 32, (2, 2), 16, 0),
    ("tf32", XPOSE_K, 32, (2, 2), XPOSE_K, 0),
    ("s8", XPOSE_K, 32, (1, 1), XPOSE_K, 0),
    ("fp8_rowwise", XPOSE_K, 32, (1, 1), XPOSE_K, 0),
    ("fp8_blockwise", XPOSE_K, 32, (1, 1), XPOSE_K, 0),    # |a b| <= 1 times scale products in {1, 2, 4}
    ("generic", GENERIC_M, 64, (2, 2), GEN_K, 0),
    ("generic_axpby", GENERIC_M, 64, (2, 2), GEN_K, 2),     # alpha = 2 (the 2 of |a b| <= 4 * 2), beta * |C| <= 1
    ("mxf4", MXF4_K + 28, 32, (1, 1), MXF4_K, 0),          # extent kpad; elements in {0, +-0.5, +-1}, quarter units
]
# growth of a partial sum beyond k |a| |b|: scale products, alpha, or the quarter units of the MXFP4 products
GRID_PRODUCT_SCALE = {"fp8_blockwise": 4, "generic_axpby": 2, "mxf4": 4}

# Group B: (name, elements of the largest buffer, footprint in bytes, k, operand magnitude)
BF16_M, BF16_N, BF16_K = 65664, 32896, 64
GRP_TOTAL_M, GRP_K, GRP_N, GRP_G = 524416, 4096, 128, 8
FP8_TOTAL_M, FP8_K, FP8_N, FP8_G = 300032, 7168, 256, 8
BAT_M, BAT_N, BAT_K, BAT_B = 32832, 32896, 64, 2
OFFSET_CASES = [
    ("bf16_c_bf16", BF16_M * BF16_N, BF16_M * BF16_N * 2 + (BF16_M + BF16_N) * BF16_K * 2, BF16_K, 2),
    ("bf16_c_f32", BF16_M * BF16_N, BF16_M * BF16_N * 4 + (BF16_M + BF16_N) * BF16_K * 2, BF16_K, 2),
    ("bf16_generic", BF16_M * BF16_N, BF16_M * BF16_N * 2 + (BF16_M * (BF16_K + 1) + BF16_N * BF16_K) * 2, BF16_K, 2),
    ("bf16_grouped", GRP_TOTAL_M * GRP_K, GRP_TOTAL_M * (GRP_K * 2 + GRP_N * 4) + GRP_G * GRP_K * GRP_N * 2, GRP_K, 2),
    ("fp8_grouped", FP8_TOTAL_M * FP8_K, FP8_TOTAL_M * (FP8_K + FP8_N * 4 + 4 * FP8_K // 128) + FP8_G * FP8_K * FP8_N,
     FP8_K, 2),
    ("bf16_batched", BAT_B * BAT_M * BAT_N, BAT_B * BAT_M * BAT_N * 2 + BAT_B * (BAT_M + BAT_N) * BAT_K * 2, BAT_K, 2),
]


def cdiv(a, b):
    return -(-a // b)


# ==== CPU: the table crosses every threshold, and every known answer is exact ========================================
def test_grid_limit_cases_cross_their_thresholds():
    names = set()
    for name, extent, tile, _, _, _ in GRID_CASES:
        names.add(name)
        blocks = cdiv(extent, tile)
        assert blocks > MAX_GRID_Y, (name, blocks)
        assert blocks < 2 * MAX_GRID_Y, (name, blocks)      # just past it: one partial second round of the grid stride
        assert extent & (extent - 1), (name, extent)        # not a power of two
    # the thresholds named in the kernels' comments
    assert cdiv(F16X2_K, 16) > MAX_GRID_Y >= cdiv(1048560, 16)
    assert cdiv(XPOSE_K, 32) > MAX_GRID_Y >= cdiv(2097120, 32)
    assert cdiv(GENERIC_M, 64) > MAX_GRID_Y >= cdiv(4194240, 64)
    kpad = cdiv(MXF4_K, 128) * 128
    assert kpad // 32 > MAX_GRID_Y and kpad == MXF4_K + 28
    assert F16X2_K % 16 and XPOSE_K % 32 and GENERIC_M % 64 and MXF4_K % 32  # a partial last block
    assert F16X2_K % 8 == 0 and XPOSE_K % 16 == 0                            # TMA-able pitches where wanted
    assert ((GEN_K + 1) * 1) % 16 and ((GEN_K + 1) * 2) % 16 and ((GEN_K + 1) * 4) % 16
    assert {"f16x2", "strict_tn", "strict_nt", "tf32", "s8", "fp8_rowwise", "fp8_blockwise", "generic", "mxf4"} <= names


def test_offset_cases_pass_2_31():
    for name, elems, footprint, _, _ in OFFSET_CASES:
        assert elems > 2 ** 31, name
        assert footprint >= elems, name
    # the grouped FP8 case: A past 2^31 bytes, with rows of the last group starting past it
    assert FP8_TOTAL_M * FP8_K > 2 ** 31 and FP8_TOTAL_M > 299593
    assert (FP8_TOTAL_M - 1) * FP8_K > 2 ** 31
    # the batched case: the last entry of C ends past 2^31 elements
    assert BAT_B * BAT_M * BAT_N > 2 ** 31


def test_known_answers_stay_below_2_24():
    for name, _, _, (ma, mb), k, extra in GRID_CASES:
        unit = GRID_PRODUCT_SCALE.get(name, 1)
        # |partial sum| in units of the smallest nonzero term, times the epilogue's growth, plus what it adds
        assert k * ma * mb * unit + extra < EXACT, name
    for name, _, _, k, mag in OFFSET_CASES:
        # 16: the FP8 cases' scale products span 1/4 .. 4, so their partial sums count quarter units up to 4 k |a| |b|
        assert k * mag * mag * 16 < EXACT, name


# ==== GPU helpers ===================================================================================================
def _gib(b):
    return f"{b / 2 ** 30:.2f} GiB"


@pytest.fixture
def free_after():
    """Every case frees what it allocated before the next one starts (the device may be shared with other work)."""
    yield
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def need(footprint):
    free, _ = torch.cuda.mem_get_info()
    if free < 1.25 * footprint:
        pytest.skip(f"needs {_gib(1.25 * footprint)} free (footprint {_gib(footprint)}), {_gib(free)} free")


def ints(shape, lo, hi, dtype, seed, chunk=1 << 26):
    """A new tensor of uniform integers in [lo, hi], generated in chunks of rows (no fp32 copy of a large operand)."""
    out = torch.empty(shape, dtype=dtype, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(seed)
    flat = out.view(-1, shape[-1])
    rows = max(1, chunk // shape[-1])
    for r0 in range(0, flat.shape[0], rows):
        part = flat[r0:r0 + rows]
        part.copy_(torch.randint(lo, hi + 1, part.shape, generator=gen, device="cuda", dtype=torch.int8))
    return out


def padded(x, pad):
    """x (rows x cols) as a view of a buffer of pitch cols + pad whose padding holds NaN (int8: 99)."""
    r, c = x.shape
    if x.dtype == torch.int8:
        buf = torch.full((r, c + pad), 99, dtype=torch.int8, device="cuda")
    elif x.dtype in (torch.float8_e4m3fn, torch.float8_e5m2):
        buf = torch.full((r, c + pad), 0x7F, dtype=torch.uint8, device="cuda").view(x.dtype)    # NaN in both formats
    else:
        buf = torch.full((r, c + pad), float("nan"), dtype=x.dtype, device="cuda")
    buf[:, :c].copy_(x)
    return buf[:, :c]


def fenced_out(rows, cols, dtype, pad=3):
    """(buffer, view): an output of pitch cols + pad, every element NaN (int32: INT32_MIN)."""
    fill = -2 ** 31 if dtype == torch.int32 else float("nan")
    buf = torch.full((rows, cols + pad), fill, dtype=dtype, device="cuda")
    return buf, buf[:, :cols]


def fence_intact(buf, cols):
    pad = buf[:, cols:]
    return bool((pad == -2 ** 31).all()) if buf.dtype == torch.int32 else bool(torch.isnan(pad.float()).all())


def check_rows(C, want_rows, chunk):
    """C (rows x n) against want_rows(r0, r1), the exact float64 rows, rounded once to C's dtype; chunk by chunk."""
    for r0 in range(0, C.shape[0], chunk):
        r1 = min(C.shape[0], r0 + chunk)
        want = want_rows(r0, r1)
        want = want.to(C.dtype) if C.dtype != torch.int32 else want.round().to(torch.int32)
        got = C[r0:r1]
        if not torch.equal(got, want):
            bad = (got != want).nonzero()[0].tolist()
            raise AssertionError(f"rows {r0}:{r1}: first difference at {bad}: got {got[bad[0], bad[1]].item()}, "
                                 f"want {want[bad[0], bad[1]].item()}")


def kchunked(a_cols, b_rows, k, chunk=1 << 19):
    """sum over K chunks of a_cols(p0, p1) @ b_rows(p0, p1) in float64: the exact product of a long-K call."""
    acc = None
    for p0 in range(0, k, chunk):
        p1 = min(k, p0 + chunk)
        t = a_cols(p0, p1) @ b_rows(p0, p1)
        acc = t if acc is None else acc + t
    return acc


def exact_small(A, B, k):
    """A (m x k) @ B (k x n) of small m and n in float64, K in chunks."""
    return kchunked(lambda p0, p1: A[:, p0:p1].double(), lambda p0, p1: B[p0:p1].double(), k)


def route(gemm, prefix):
    assert gemm.last_kernel().startswith(prefix), (gemm.last_kernel(), prefix)


# ==== A. grid limits: F16X2 (col_absmax_kernel, rows = k) ===========================================================
@gpu
@pytest.mark.parametrize("case", ["nn", "tn_python", "auto", "packed_b"])
def test_f16x2_long_k(gemm, hooks, free_after, case):
    m = n = 64
    k = F16X2_K
    A = padded(ints((m, k), -2, 2, torch.float32, 1), 8)
    B = padded(ints((k, n), -2, 2, torch.float32, 2), 8)
    buf, C = fenced_out(m, n, torch.float32, pad=4)
    l0 = gemm.launch_count()
    if case == "nn":
        gemm.gemm_f32(A, B, out=C, mode=gemm.F32_F16X2)
    elif case == "tn_python":             # dW = x^T dy: A given as x.t(), B row-major; both split by column maxima
        x = padded(A.t().contiguous(), 8)
        gemm.gemm(x.t(), B, out=C)
    elif case == "auto":
        gemm.gemm_f32(A, B, out=C, mode=gemm.F32_AUTO)
    else:
        pb = gemm.PackedB(B, mode=gemm.F32_F16X2)
        gemm.gemm_f32_packed(A, pb, out=C)
        pb.close()
    route(gemm, "tc_f16x2")
    assert gemm.launch_count() - l0 >= 2
    torch.cuda.synchronize()
    assert torch.equal(C.double(), exact_small(A, B, k))
    assert fence_intact(buf, n)


# ==== A. grid limits: transposes (transpose_kernel, rows = k or n) ==================================================
@gpu
@pytest.mark.parametrize("lay", ["tn", "nt"])
def test_strict_transposed_operands(gemm, hooks, free_after, lay):
    m = 64
    if lay == "tn":                       # A given as A^T (k x m): rows = k
        n, k = 64, XPOSE_K
        x = padded(ints((k, m), -2, 2, torch.float32, 3), 4)
        B = padded(ints((k, n), -2, 2, torch.float32, 4), 4)
        A = x.t()
        want = lambda r0, r1: exact_small(x.t()[r0:r1], B, k)
    else:                                 # B given as B^T (n x k): rows = n
        n, k = XPOSE_K, 16
        A = padded(ints((m, k), -2, 2, torch.float32, 5), 4)
        W = padded(ints((n, k), -2, 2, torch.float32, 6), 4)
        B = W.t()
        want = lambda r0, r1: A[r0:r1].double() @ W.double().t()
    buf, C = fenced_out(m, n, torch.float32)
    gemm.gemm(A, B, out=C, mode=gemm.F32_STRICT)
    route(gemm, "ffma")
    check_rows(C, want, 64)
    assert fence_intact(buf, n)


@gpu
def test_tf32_row_major_b(gemm, hooks, free_after):
    m = n = 64
    k = XPOSE_K
    A = padded(ints((m, k), -2, 2, torch.float32, 7), 4)
    B = padded(ints((k, n), -2, 2, torch.float32, 8), 4)
    buf, C = fenced_out(m, n, torch.float32)
    gemm.gemm_f32(A, B, out=C, mode=gemm.F32_TF32)
    route(gemm, "tc_tf32")
    assert torch.equal(C.double(), exact_small(A, B, k))
    assert fence_intact(buf, n)


@gpu
@pytest.mark.parametrize("case", ["s8s32", "requant", "s8s32_nt_in_place"])
def test_int8_long_k(gemm, oracle, hooks, free_after, case):
    m = n = 64
    k = XPOSE_K
    A = padded(ints((m, k), -1, 1, torch.int8, 9), 16)
    if case == "s8s32_nt_in_place":       # control: B^T is read in place, no transpose
        W = padded(ints((n, k), -1, 1, torch.int8, 10), 16)
        B, Bd = W.t(), W.t()
    else:
        B = padded(ints((k, n), -1, 1, torch.int8, 10), 16)
        Bd = B
    exact = exact_small(A, Bd, k)
    if case == "requant":
        scales = torch.tensor([2.0 ** -(i % 9) for i in range(m)], dtype=torch.float32, device="cuda")
        buf = torch.full((m, n + 16), 77, dtype=torch.int8, device="cuda")
        C = buf[:, :n]
        gemm.gemm_s8s8_requant(A, B, scales, out=C)
        route(gemm, "tc_s8_requant")
        want = _libs.requant_s8(oracle, exact.round().to(torch.int32).cpu().numpy(), scales.cpu().numpy())
        assert np.array_equal(C.cpu().numpy(), want)
        assert bool((buf[:, n:] == 77).all())
        return
    buf, C = fenced_out(m, n, torch.int32)
    gemm.gemm(A, B, out=C)
    route(gemm, "tc_s8")
    assert torch.equal(C, exact.round().to(torch.int32))
    assert fence_intact(buf, n)


@gpu
@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_16bit_long_k_in_place(gemm, hooks, free_after, dtype):
    """Controls at the transposes' K: 16-bit operands are read in place in either layout."""
    dt = getattr(torch, dtype)
    m = n = 64
    k = XPOSE_K
    A = padded(ints((m, k), -2, 2, dt, 11), 8)
    B = padded(ints((k, n), -2, 2, dt, 12), 8)
    buf, C = fenced_out(m, n, torch.float32)
    gemm.gemm(A, B, out=C)
    route(gemm, "tc_bf16" if dtype == "bfloat16" else "tc_f16")
    assert torch.equal(C.double(), exact_small(A, B, k))
    assert fence_intact(buf, n)


def _fp8_operands(m, n, k, lay, seed):
    """(A, B, A64, B64): FP8 e4m3 operands in [-1, 1] as the call sees them (lay 'nn': row-major B, transposed in the
    workspace; 'tn': A given as A^T, B column-major) and their float64 values as row-major m x k / k x n."""
    f8 = torch.float8_e4m3fn
    if lay == "nn":
        A = padded(ints((m, k), -1, 1, torch.float32, seed).to(f8), 16)
        B = padded(ints((k, n), -1, 1, torch.float32, seed + 1).to(f8), 16)
        return A, B, A.float(), B.float()
    x = padded(ints((k, m), -1, 1, torch.float32, seed).to(f8), 16)
    W = padded(ints((n, k), -1, 1, torch.float32, seed + 1).to(f8), 16)
    return x.t(), W.t(), x.float().t(), W.float().t()


@gpu
@pytest.mark.parametrize("lay", ["nn", "tn"])
@pytest.mark.parametrize("recipe", ["rowwise", "blockwise"])
def test_fp8_transposed_long_k(gemm, hooks, free_after, lay, recipe):
    m = n = 64
    k = XPOSE_K
    A, B, Ad, Bd = _fp8_operands(m, n, k, lay, 13)
    gen = torch.Generator(device="cuda").manual_seed(14)
    buf, C = fenced_out(m, n, torch.float32)
    if recipe == "rowwise":
        sa = (2.0 ** torch.randint(-1, 2, (m, 1), generator=gen, device="cuda")).float()
        sb = (2.0 ** torch.randint(-1, 2, (1, n), generator=gen, device="cuda")).float()
        gemm.scaled_mm(A, B, sa, sb, out_dtype=torch.float32, out=C)
        want = exact_small(Ad, Bd, k) * sa.double() * sb.double()
    else:                                 # 1 x 128 A, 128 x 128 B; scales in {1, 2}
        q = cdiv(k, 128)
        sa = (2.0 ** torch.randint(0, 2, (m, q), generator=gen, device="cuda")).float()
        sb = (2.0 ** torch.randint(0, 2, (q, cdiv(n, 128)), generator=gen, device="cuda")).float()
        gemm.scaled_mm(A, B, sa, sb, out_dtype=torch.float32, out=C)
        col_blk = torch.arange(n, device="cuda") // 128
        want = kchunked(lambda p0, p1: Ad[:, p0:p1].double() * sa.double()[:, torch.arange(p0, p1, device="cuda") // 128],
                        lambda p0, p1: Bd[p0:p1].double() * sb.double()[torch.arange(p0, p1, device="cuda") // 128][:, col_blk],
                        k)
    route(gemm, "tc_e4m3_")
    assert torch.equal(C.double(), want)
    assert fence_intact(buf, n)


# ==== A. grid limits: the generic CUDA-core kernels (ceil(m / 64) row blocks) =======================================
def _generic_operands(dt, seed, batch=None):
    """A (m x GEN_K) at pitch GEN_K + 1 (no operand type can use TMA) with NaN padding, B (GEN_K x GEN_N) row-major."""
    m, k, n = GENERIC_M, GEN_K, GEN_N
    if batch is None:
        A = padded(ints((m, k), -2 if dt != torch.int8 else -1, 2 if dt != torch.int8 else 1, dt, seed), 1)
        B = ints((k, n), -2 if dt != torch.int8 else -1, 2 if dt != torch.int8 else 1, dt, seed + 1)
        return A, B
    abuf = torch.full((batch, m, k + 1), float("nan"), dtype=dt, device="cuda")
    for b in range(batch):
        abuf[b, :, :k].copy_(ints((m, k), -2, 2, dt, seed + 2 * b))
    B = torch.stack([ints((k, n), -2, 2, dt, seed + 2 * b + 1) for b in range(batch)])
    return abuf[:, :, :k], B


CHUNK = 1 << 20


@gpu
@pytest.mark.parametrize("mode", ["F32_STRICT", "F32_TF32"])
def test_generic_f32_tall_m(gemm, hooks, free_after, mode):
    A, B = _generic_operands(torch.float32, 21)
    buf, C = fenced_out(GENERIC_M, GEN_N, torch.float32)
    gemm.gemm(A, B, out=C, mode=getattr(gemm, mode))
    route(gemm, "generic_f32_64x64")
    check_rows(C, lambda r0, r1: A[r0:r1].double() @ B.double(), CHUNK)
    assert fence_intact(buf, GEN_N)


@gpu
@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
@pytest.mark.parametrize("c16", [False, True])
def test_generic_16bit_tall_m_alpha_beta(gemm, hooks, free_after, dtype, c16):
    dt = getattr(torch, dtype)
    A, B = _generic_operands(dt, 23)
    cdt = dt if c16 else torch.float32
    buf, C = fenced_out(GENERIC_M, GEN_N, cdt)
    C0 = ints((GENERIC_M, GEN_N), -2, 2, cdt, 25)
    C.copy_(C0)
    gemm.gemm(A, B, out=C, alpha=2.0, beta=0.5)
    route(gemm, "generic_" + ("bf16" if dtype == "bfloat16" else "f16") + "_64x64")
    check_rows(C, lambda r0, r1: 2.0 * (A[r0:r1].double() @ B.double()) + 0.5 * C0[r0:r1].double(), CHUNK)
    assert fence_intact(buf, GEN_N)


@gpu
def test_generic_bf16_tall_m_bias_gelu(gemm, hooks, free_after):
    """GELU has no exact float64 restatement here: the tall call must equal the same call made in two halves, each
    under the old limit (same kernel, same arithmetic per element)."""
    A, B = _generic_operands(torch.bfloat16, 27)
    bias = ints((GEN_N,), -2, 2, torch.bfloat16, 28)
    buf, C = fenced_out(GENERIC_M, GEN_N, torch.bfloat16)
    gemm.gemm(A, B, out=C, bias=bias, activation="gelu", out_dtype=torch.bfloat16)
    route(gemm, "generic_bf16_64x64")
    half = 1 << 21
    _, W = fenced_out(GENERIC_M, GEN_N, torch.bfloat16)
    gemm.gemm(A[:half], B, out=W[:half], bias=bias, activation="gelu", out_dtype=torch.bfloat16)
    gemm.gemm(A[half:], B, out=W[half:], bias=bias, activation="gelu", out_dtype=torch.bfloat16)
    route(gemm, "generic_bf16_64x64")
    assert not torch.isnan(W.float()).any()
    for r0 in range(0, GENERIC_M, CHUNK):
        assert torch.equal(C[r0:r0 + CHUNK].view(torch.int16), W[r0:r0 + CHUNK].view(torch.int16)), r0
    assert fence_intact(buf, GEN_N)


@gpu
def test_generic_s8s32_tall_m(gemm, hooks, free_after):
    A, B = _generic_operands(torch.int8, 29)
    buf, C = fenced_out(GENERIC_M, GEN_N, torch.int32)
    gemm.gemm(A, B, out=C)
    route(gemm, "generic_s8_64x64")
    check_rows(C, lambda r0, r1: A[r0:r1].double() @ B.double(), CHUNK)
    assert fence_intact(buf, GEN_N)


@gpu
@pytest.mark.parametrize("k0", [False, True])
def test_generic_requant_tall_m(gemm, oracle, hooks, free_after, k0):
    A, B = _generic_operands(torch.int8, 31)
    if k0:                                # the k == 0 path: C = requant(0) per row
        A, B = A[:, :0], B[:0]
    m = GENERIC_M
    scales = (2.0 ** -torch.randint(0, 4, (m,), device="cuda")).float()
    bias = ints((m,), -3, 3, torch.float32, 33)
    buf = torch.full((m, GEN_N + 3), 77, dtype=torch.int8, device="cuda")
    C = buf[:, :GEN_N]
    gemm.gemm_s8s8_requant(A, B, scales, bias=bias, out=C)
    route(gemm, "generic_s8_requant_64x64")
    for r0 in range(0, m, CHUNK):
        r1 = min(m, r0 + CHUNK)
        c32 = (A[r0:r1].double() @ B.double()).round().to(torch.int32) if not k0 else \
            torch.zeros((r1 - r0, GEN_N), dtype=torch.int32, device="cuda")
        want = _libs.requant_s8(oracle, c32.cpu().numpy(), scales[r0:r1].cpu().numpy(), bias[r0:r1].cpu().numpy())
        assert np.array_equal(C[r0:r1].cpu().numpy(), want), r0
    assert bool((buf[:, GEN_N:] == 77).all())


@gpu
def test_generic_batched_tall_m(gemm, hooks, free_after):
    A, B = _generic_operands(torch.bfloat16, 35, batch=2)
    buf = torch.full((2, GENERIC_M, GEN_N + 3), float("nan"), dtype=torch.bfloat16, device="cuda")
    C = buf[:, :, :GEN_N]
    gemm.gemm(A, B, out=C, out_dtype=torch.bfloat16)
    route(gemm, "generic_bf16_bat_64x64")
    for b in range(2):
        check_rows(C[b], lambda r0, r1: A[b, r0:r1].double() @ B[b].double(), CHUNK)
    assert bool(torch.isnan(buf[:, :, GEN_N:].float()).all())


@gpu
def test_generic_grouped_controls_tall(gemm, hooks, free_after):
    """Controls: the grouped generic kernel at the same total M and the K-grouped one at the same total K."""
    A, _ = _generic_operands(torch.bfloat16, 37)
    B3 = torch.stack([ints((GEN_K, GEN_N), -2, 2, torch.bfloat16, 38 + g) for g in range(2)])
    ends = [GENERIC_M // 3, GENERIC_M]
    offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
    buf, C = fenced_out(GENERIC_M, GEN_N, torch.float32)
    gemm.gemm(A, B3, out=C, offs=offs)
    route(gemm, "generic_bf16_grp_64x64")
    g_of = lambda r0, r1: [(max(r0, s), min(r1, e), g) for g, (s, e) in enumerate(zip([0] + ends[:-1], ends))
                           if max(r0, s) < min(r1, e)]
    check_rows(C, lambda r0, r1: torch.cat([A[s:e].double() @ B3[g].double() for s, e, g in g_of(r0, r1)]), CHUNK)
    assert fence_intact(buf, GEN_N)
    del C, buf
    # K-grouped: dW_g = dy_g^T x_g over total_k = GENERIC_M rows, dy read as a transposed view of pitch m + 1
    m, n = 40, 24
    dy = padded(ints((GENERIC_M, m), -2, 2, torch.bfloat16, 41), 1)
    x = ints((GENERIC_M, n), -2, 2, torch.bfloat16, 42)
    out = torch.full((2, m, n), float("nan"), dtype=torch.float32, device="cuda")
    gemm.gemm(dy.t(), x, out=out, offs=offs)
    route(gemm, "generic_bf16_kgrp_64x64")
    for g, (s, e) in enumerate(zip([0] + ends[:-1], ends)):
        want = kchunked(lambda p0, p1: dy[s + p0:s + p1].double().t(), lambda p0, p1: x[s + p0:s + p1].double(), e - s)
        assert torch.equal(out[g].double(), want), g


# ==== A. grid limits: MXFP4 (kpad / 32 K-blocks) ====================================================================
@gpu
def test_mxf4_long_k(gemm, oracle, hooks, free_after):
    import test_mxf4 as mx
    o = mx._o(oracle)
    m = n = 32
    k = MXF4_K
    rng = np.random.default_rng(43)
    grid = np.array([0, .5, 1, -.5, -1], np.float32)    # with a 1 in every 32-block: scale 2^-2, codes exact

    def operand(rows):
        x = rng.choice(grid, (rows, k)).astype(np.float32)
        x[:, ::32] = 1.0
        return x
    a, bt = operand(m), operand(n)                     # bt = B^T (n x k)
    qb_ref, sb_ref, kpad = mx.quant(o, bt)
    qa_ref, sa_ref, _ = mx.quant(o, a)
    B = torch.from_numpy(np.ascontiguousarray(bt.T)).cuda()
    qb, sfb, rows, kk = gemm.mxf4_quantize(B, transpose=True)
    assert (rows, kk) == (n, k) and gemm.last_kernel() == "mxf4_quantize_cols_t"
    assert np.array_equal(qb.cpu().numpy().reshape(n, kpad // 2), qb_ref)
    assert np.array_equal(sfb.cpu().numpy(), mx.atoms(o, sb_ref, n, kpad))
    del B
    qa, sfa, _, _ = gemm.mxf4_quantize(torch.from_numpy(a).cuda())
    buf, C = fenced_out(m, n, torch.float32)
    gemm.gemm_mxf4(qa, sfa, qb, sfb, m, n, k, out=C)
    assert gemm.last_kernel() == "tc_mxf4_128x128"
    assert np.array_equal(C.cpu().numpy().astype(np.float64), a.astype(np.float64) @ bt.astype(np.float64).T)
    assert fence_intact(buf, n)


# ==== B. 64-bit offsets =============================================================================================
def _footprint(name):
    return next(f for nm, _, f, _, _ in OFFSET_CASES if nm == name)


@gpu
@pytest.mark.parametrize("case", ["bf16_c_bf16", "bf16_c_f32", "bf16_generic"])
def test_bf16_c_past_2_31(gemm, hooks, free_after, case):
    need(_footprint(case))
    m, n, k = BF16_M, BF16_N, BF16_K
    A = ints((m, k), -2, 2, torch.bfloat16, 51)
    if case == "bf16_generic":
        A = padded(A, 1)
    B = ints((k, n), -2, 2, torch.bfloat16, 52)
    cdt = torch.float32 if case == "bf16_c_f32" else torch.bfloat16
    C = torch.full((m, n), float("nan"), dtype=cdt, device="cuda")
    gemm.gemm(A, B, out=C)
    route(gemm, "generic_bf16_64x64" if case == "bf16_generic" else "tc_bf16")
    check_rows(C, lambda r0, r1: A[r0:r1].double() @ B.double(), 4096)


@gpu
def test_grouped_bf16_a_past_2_31(gemm, hooks, free_after):
    need(_footprint("bf16_grouped"))
    total_m, k, n, G = GRP_TOTAL_M, GRP_K, GRP_N, GRP_G
    A = ints((total_m, k), -2, 2, torch.bfloat16, 53)
    W = ints((G, n, k), -2, 2, torch.bfloat16, 54)
    ends = [total_m * (g + 1) // G - (37 if g < G - 1 else 0) for g in range(G)]
    offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
    C = torch.full((total_m, n), float("nan"), dtype=torch.float32, device="cuda")
    gemm.gemm(A, W.transpose(-2, -1), out=C, offs=offs)
    route(gemm, "tc_bf16")
    for g, (s, e) in enumerate(zip([0] + ends[:-1], ends)):
        check_rows(C[s:e], lambda r0, r1: A[s + r0:s + r1].double() @ W[g].double().t(), 8192)


def _fp8_grouped_operands(seed):
    total_m, k, n, G = FP8_TOTAL_M, FP8_K, FP8_N, FP8_G
    f8 = torch.float8_e4m3fn
    A = torch.empty((total_m, k), dtype=f8, device="cuda")
    for r0 in range(0, total_m, 8192):
        A[r0:r0 + 8192].copy_(ints((min(8192, total_m - r0), k), -2, 2, torch.float32, seed + r0))
    W = ints((G, n, k), -2, 2, torch.float32, seed - 1).to(f8)
    ends = [total_m * (g + 1) // G - (53 if g < G - 1 else 0) for g in range(G)]
    return A, W, ends


@gpu
@pytest.mark.parametrize("recipe", ["rowwise", "blockwise", "blockwise_fp8_out"])
def test_grouped_fp8_a_past_2_31_bytes(gemm, hooks, free_after, recipe):
    need(_footprint("fp8_grouped"))
    total_m, k, n, G = FP8_TOTAL_M, FP8_K, FP8_N, FP8_G
    A, W, ends = _fp8_grouped_operands(61)
    offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(62)
    q = k // 128
    spans = list(zip([0] + ends[:-1], ends))
    if recipe == "rowwise":
        sa = (2.0 ** torch.randint(-1, 2, (total_m,), generator=gen, device="cuda")).float()
        sb = (2.0 ** torch.randint(-1, 2, (G, n), generator=gen, device="cuda")).float()
    else:
        sa = (2.0 ** torch.randint(-1, 2, (total_m, q), generator=gen, device="cuda")).float()
        sb = (2.0 ** torch.randint(-1, 2, (G, q, cdiv(n, 128)), generator=gen, device="cuda")).float()
    if recipe == "blockwise_fp8_out":
        # each group must be bit for bit the single-matrix call on its own rows (offsets below 2^31 there)
        C, sc = gemm.scaled_grouped_mm_quant(A, W.transpose(-2, -1), sa, sb, offs=offs)
        name = gemm.last_kernel()
        for g, (s, e) in enumerate(spans):
            c1, s1 = gemm.scaled_mm_quant(A[s:e], W[g].t(), sa[s:e], sb[g])
            assert torch.equal(C[s:e].view(torch.uint8), c1.view(torch.uint8)), g
            assert torch.equal(sc[s:e], s1), g
        assert name.startswith("tc_e4m3_oe4m3_grp"), name
        return
    C = torch.full((total_m, n), float("nan"), dtype=torch.float32, device="cuda")
    gemm.scaled_grouped_mm(A, W.transpose(-2, -1), sa, sb, offs=offs, out_dtype=torch.float32, out=C)
    assert gemm.last_kernel().startswith("tc_e4m3_of32_grp"), gemm.last_kernel()
    for g, (s, e) in enumerate(spans):
        if recipe == "rowwise":
            want = lambda r0, r1: (A[s + r0:s + r1].float().double() @ W[g].float().double().t()) * \
                sa[s + r0:s + r1, None].double() * sb[g].double()
        else:
            cb = torch.arange(n, device="cuda") // 128
            kb = torch.arange(k, device="cuda") // 128
            want = lambda r0, r1: (A[s + r0:s + r1].float().double() * sa[s + r0:s + r1][:, kb].double()) @ \
                (W[g].float().double().t() * sb[g].double()[kb][:, cb])
        check_rows(C[s:e], want, 8192)
    assert bool(torch.isnan(C[ends[-1]:]).all())


@gpu
def test_batched_bf16_c_past_2_31(gemm, hooks, free_after):
    need(_footprint("bf16_batched"))
    A = ints((BAT_B, BAT_M, BAT_K), -2, 2, torch.bfloat16, 71)
    B = ints((BAT_B, BAT_K, BAT_N), -2, 2, torch.bfloat16, 72)
    C = torch.full((BAT_B, BAT_M, BAT_N), float("nan"), dtype=torch.bfloat16, device="cuda")
    gemm.gemm(A, B, out=C, out_dtype=torch.bfloat16)
    route(gemm, "tc_bf16")
    for b in range(BAT_B):
        check_rows(C[b], lambda r0, r1: A[b, r0:r1].double() @ B[b].double(), 4096)
