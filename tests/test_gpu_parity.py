"""Parity tests proper (-m gpu): the CUDA path through the C ABI against the oracle, the committed
golden vectors of the reference, and size-independent properties at BASELINE.json's full sizes.

Bars: bit-exact for int8->int32 and for the strict fp32 path (sequential-k FFMA == the reference's
naive REF_MMult as its own flags build it); tensor-core fp32/bf16 within the north_star tolerance
1e-3 * max|Cref| (tightened per mode below)."""
import os

import numpy as np
import pytest

import _libs

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_vectors.npz"))
TOL_TF32 = 1e-3     # north_star: within 1e-3 max relative error of REF_MMult
TOL_BF16 = 2e-5     # bf16-rounded inputs, fp32 accumulate: only accumulation-order noise remains


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def rel(c, t):
    return float(np.abs(c.astype(np.float64) - t).max() / max(np.abs(t).max(), 1e-30))


SHAPES = [(1, 1, 1), (4, 4, 4), (7, 9, 5), (64, 48, 80), (77, 77, 77), (128, 128, 128), (128, 256, 64),
          (130, 70, 257), (256, 384, 512), (300, 260, 100), (1, 1000, 333), (1000, 1, 77), (513, 1027, 260)]


@pytest.mark.parametrize("m,n,k", SHAPES)
def test_f32_strict_bit_exact(gemm, oracle, m, n, k):
    a, b = _libs.gen_f32(oracle, m, k, 21), _libs.gen_f32(oracle, k, n, 22)
    c = gemm.gemm_f32(cuda(a), cuda(b), mode=gemm.F32_STRICT).cpu().numpy()
    assert np.array_equal(c, _libs.ref_f32_fma(oracle, a, b)), gemm.last_kernel()


@pytest.mark.parametrize("pad_a,pad_b,pad_c", [(0, 0, 0), (4, 8, 12), (1, 0, 0), (0, 3, 0), (0, 0, 5), (3, 5, 7)])
def test_f32_strict_leading_dimensions(gemm, oracle, pad_a, pad_b, pad_c):
    """lda/ldb/ldc != k/n/n: the reference never exercises these (cuda/test_MMult.cpp:62) and its
    kernels ignore them; the C ABI honours them, aligned (TMA) or not (generic kernel)."""
    m, n, k = 200, 136, 264
    A = cuda(_libs.gen_f32(oracle, m, k + pad_a, 1))[:, :k]
    B = cuda(_libs.gen_f32(oracle, k, n + pad_b, 2))[:, :n]
    Cbuf = torch.full((m, n + pad_c), -7.0, device="cuda")
    gemm.gemm_f32(A, B, out=Cbuf[:, :n], mode=gemm.F32_STRICT)
    ref = _libs.ref_f32_fma(oracle, A.cpu().numpy(), B.cpu().numpy())
    assert np.array_equal(Cbuf[:, :n].cpu().numpy(), ref), gemm.last_kernel()
    if pad_c:
        assert (Cbuf[:, n:] == -7.0).all(), "wrote outside the m x n window"


@pytest.mark.parametrize("m,n,k", SHAPES)
def test_f32_tf32_within_tolerance(gemm, oracle, m, n, k):
    a, b = _libs.gen_f32(oracle, m, k, 23), _libs.gen_f32(oracle, k, n, 24)
    c = gemm.gemm_f32(cuda(a), cuda(b), mode=gemm.F32_TF32).cpu().numpy()
    t = _libs.ref_f64(oracle, a, b)
    assert rel(c, t) <= TOL_TF32, (gemm.last_kernel(), rel(c, t))
    # and under the reference harness's own gate (cuda/test_MMult.cpp:124)
    assert np.abs(c - _libs.ref_f32_fma(oracle, a, b)).max() < 0.5


TOL_X3 = 1e-5      # split-bf16 x3 with two-level accumulation: fp32-class (strict FFMA measures ~3e-6 at K=4096)
TOL_X2 = 4e-5      # split-bf16 x2: dropped a2*b2 term, ~2^-17 relative


TOL_F16X2 = 1e-5   # scaled split-fp16, 22-bit operands: normwise fp32-class


@pytest.mark.parametrize("m,n,k", SHAPES + [(1000, 1100, 4096), (260, 200, 1500)])
def test_f32_split_f16_scaled(gemm, oracle, m, n, k):
    a, b = _libs.gen_f32(oracle, m, k, 35), _libs.gen_f32(oracle, k, n, 36)
    c = gemm.gemm_f32(cuda(a), cuda(b), mode=gemm.F32_F16X2).cpu().numpy()
    assert gemm.last_kernel().startswith("tc_f16x2"), gemm.last_kernel()
    t = _libs.ref_f64(oracle, a, b)
    assert rel(c, t) <= TOL_F16X2, (gemm.last_kernel(), rel(c, t))


def test_f32_split_f16_dynamic_range(gemm, oracle):
    """fp16 has 5 exponent bits: the mode must survive rows of A / columns of B spread over 2^+-20
    (power-of-two row/column scaling is exact, so the scaled result must track the unscaled one)."""
    m, n, k = 384, 520, 1024
    rng = np.random.default_rng(7)
    a0, b0 = _libs.gen_f32(oracle, m, k, 37), _libs.gen_f32(oracle, k, n, 38)
    rs = np.exp2(rng.integers(-20, 21, m)).astype(np.float32)
    cs = np.exp2(rng.integers(-20, 21, n)).astype(np.float32)
    rs[5], cs[7] = 0.0, 0.0                                   # an all-zero row and column
    a, b = a0 * rs[:, None], b0 * cs[None, :]
    c = gemm.gemm_f32(cuda(a), cuda(b), mode=gemm.F32_F16X2).cpu().numpy()
    t = _libs.ref_f64(oracle, a, b)
    scale = rs[:, None].astype(np.float64) * cs[None, :]
    ok = scale > 0
    err = np.abs(c - t)[ok] / scale[ok]
    assert err.max() <= TOL_F16X2 * np.abs(_libs.ref_f64(oracle, a0, b0)).max()
    assert (c[~ok] == 0).all() and np.isfinite(c).all()
    ones = torch.ones((300, 300), device="cuda")
    assert (gemm.gemm_f32(ones * 3, ones, mode=gemm.F32_F16X2) == 900).all()


@pytest.mark.parametrize("m,n,k", SHAPES + [(1000, 1100, 4096), (260, 200, 1500)])
@pytest.mark.parametrize("mode,tol", [("x3", TOL_X3), ("x2", TOL_X2)])
def test_f32_split_bf16_modes(gemm, oracle, m, n, k, mode, tol):
    """fp32 in / fp32 out on the tensor cores: bf16 planes (exact split of the fp32 inputs), every
    significant cross term, K folded in chunks.  Also inside the reference harness's own 0.5 gate."""
    md = gemm.F32_BF16X3 if mode == "x3" else gemm.F32_BF16X2
    a, b = _libs.gen_f32(oracle, m, k, 33), _libs.gen_f32(oracle, k, n, 34)
    c = gemm.gemm_f32(cuda(a), cuda(b), mode=md).cpu().numpy()
    assert gemm.last_kernel().startswith("tc_bf16" + mode), gemm.last_kernel()
    t = _libs.ref_f64(oracle, a, b)
    assert rel(c, t) <= tol, (gemm.last_kernel(), rel(c, t))
    assert np.abs(c - _libs.ref_f32_fma(oracle, a, b)).max() < 1e-2


def test_f32_split_unaligned_and_default(gemm, oracle):
    """The split pre-pass reads fp32 through plain loads, so odd leading dimensions still take the
    tensor-core path; AUTO resolves to F16X2 (include/b200gemm.h)."""
    m, n, k = 200, 136, 264
    A = cuda(_libs.gen_f32(oracle, m, k + 3, 1))[:, :k]
    B = cuda(_libs.gen_f32(oracle, k, n + 5, 2))[:, :n]
    Cbuf = torch.full((m, n + 7), -7.0, device="cuda")
    assert gemm.lib.b200_gemm_default_f32_mode() == gemm.F32_F16X2 or os.environ.get("B200GEMM_F32_MODE")
    gemm.gemm_f32(A, B, out=Cbuf[:, :n], mode=gemm.F32_BF16X3)
    assert gemm.last_kernel().startswith("tc_bf16x3")
    t = _libs.ref_f64(oracle, A.cpu().numpy(), B.cpu().numpy())
    assert rel(Cbuf[:, :n].cpu().numpy(), t) <= TOL_X3
    assert (Cbuf[:, n:] == -7.0).all()
    # exactly representable inputs: every mode must be exact (ones fixture of the aarch64 harness)
    ones = torch.ones((300, 300), device="cuda")
    for md in (gemm.F32_BF16X3, gemm.F32_BF16X2):
        assert (gemm.gemm_f32(ones, ones, mode=md) == 300).all()


@pytest.mark.parametrize("m,n,k", SHAPES)
@pytest.mark.parametrize("out", ["f32", "bf16"])
def test_bf16(gemm, oracle, m, n, k, out):
    a = _libs.round_bf16(oracle, _libs.gen_f32(oracle, m, k, 25))
    b = _libs.round_bf16(oracle, _libs.gen_f32(oracle, k, n, 26))
    od = torch.float32 if out == "f32" else torch.bfloat16
    c = gemm.gemm_bf16(cuda(a).bfloat16(), cuda(b).bfloat16(), out_dtype=od).float().cpu().numpy()
    t = _libs.ref_f64(oracle, a, b)
    if out == "f32":
        assert rel(c, t) <= TOL_BF16, (gemm.last_kernel(), rel(c, t))
    else:   # one RNE rounding of the fp32 accumulator to bf16: half an ulp = 2^-9 relative, elementwise
        assert np.all(np.abs(c - t) <= np.abs(t) * 2.0 ** -8 + TOL_BF16 * np.abs(t).max())


@pytest.mark.parametrize("m,n,k", SHAPES + [(128, 256, 4096), (33, 47, 1000)])
def test_s8s32_bit_exact(gemm, oracle, m, n, k):
    a, b = _libs.gen_s8(oracle, m, k, 27), _libs.gen_s8(oracle, k, n, 28)
    c = gemm.gemm_s8s32(cuda(a), cuda(b)).cpu().numpy()
    assert np.array_equal(c, _libs.ref_s8(oracle, a, b)), gemm.last_kernel()


def test_s8_extremes_and_alignment(gemm, oracle):
    """[-127,127] extremes (chgemm input contract, /root/reference/README.md:82); 16-byte aligned
    pitches go through the int8 wgmma kernel, everything else through the CUDA-core kernel: same bits."""
    m, n, k = 160, 272, 512
    for fill_a, fill_b in [(127, 127), (-127, 127), (-127, -127)]:
        a = np.full((m, k), fill_a, np.int8)
        b = np.full((k, n), fill_b, np.int8)
        c = gemm.gemm_s8s32(cuda(a), cuda(b)).cpu().numpy()
        assert gemm.last_kernel().startswith("tc_s8")
        assert (c == fill_a * fill_b * k).all()
    a, b = _libs.gen_s8(oracle, m, k + 16, 1), _libs.gen_s8(oracle, k + 16, n + 16, 2)
    A, B = cuda(a), cuda(b)
    c_tc = gemm.gemm_s8s32(A[:, :k], B[:k, :n]).cpu().numpy()
    k_tc = gemm.last_kernel()
    c_cc = gemm.gemm_s8s32(A[:, 1:k + 1], B[1:k + 1, 1:n + 1]).cpu().numpy()   # misaligned bases
    assert k_tc.startswith("tc_s8") and gemm.last_kernel().startswith("generic_s8")
    assert np.array_equal(c_tc, _libs.ref_s8(oracle, a[:, :k], b[:k, :n]))
    assert np.array_equal(c_cc, _libs.ref_s8(oracle, a[:, 1:k + 1], b[1:k + 1, 1:n + 1]))


def _rq_case(oracle, m, n, k, seed, kind):
    a, b = _libs.gen_s8(oracle, m, k, seed), _libs.gen_s8(oracle, k, n, seed + 1)
    rng = np.random.default_rng(seed)
    if kind == "ties":          # power-of-two scales: every odd accumulator lands exactly on a .5 tie
        scales = np.float32(2.0) ** -rng.integers(1, 9, m).astype(np.float32)
        bias = (rng.integers(-8, 9, m) * 0.5).astype(np.float32)
    elif kind == "saturate":    # most products leave [-128, 127]
        scales = rng.uniform(0.01, 0.5, m).astype(np.float32)
        bias = rng.uniform(-300, 300, m).astype(np.float32)
    else:                       # what a quantised layer passes: |acc| ~ 127^2 sqrt(k) / 3 mapped to ~[-100, 100]
        scales = (rng.uniform(0.5, 2.0, m) * 300.0 / (127.0 ** 2 * max(k, 1) ** 0.5)).astype(np.float32)
        bias = rng.uniform(-20, 20, m).astype(np.float32)
    return a, b, scales, bias


@pytest.mark.parametrize("kind", ["ties", "saturate", "layer"])
@pytest.mark.parametrize("m,n,k", [(128, 128, 64), (300, 528, 208), (77, 96, 80), (512, 1024, 1024),
                                   (1000, 1104, 2048), (2304, 2304, 512)])
def test_s8_requant_bit_exact(gemm, oracle, m, n, k, kind):
    """int8 out through the fused requant epilogue == oracle_requant(REF_MMult int32) bit for bit
    (aarch64-int8/int8kernel_m4.S:386-426), with and without bias, tensor-core and generic paths."""
    a, b, scales, bias = _rq_case(oracle, m, n, k, 61, kind)
    c32 = _libs.ref_s8(oracle, a, b)
    A, B, S, Bi = cuda(a), cuda(b), cuda(scales), cuda(bias)
    out = gemm.gemm_s8s8_requant(A, B, S, Bi).cpu().numpy()
    assert gemm.last_kernel().startswith("tc_s8_requant"), gemm.last_kernel()
    assert np.array_equal(out, _libs.requant_s8(oracle, c32, scales, bias))
    out = gemm.gemm_s8s8_requant(A, B, S, None).cpu().numpy()            # bias == NULL (cmp bias, #0)
    assert np.array_equal(out, _libs.requant_s8(oracle, c32, scales, None))
    if kind == "ties":
        assert (out != np.clip(np.rint(c32 * scales[:, None]), -128, 127)).any()   # ties-to-even would differ


def test_s8_requant_generic_path_and_edges(gemm, oracle):
    m, n, k = 130, 208, 112            # + 16: pitches 224 and 128 bytes, TMA-able when the base is aligned
    a, b, scales, bias = _rq_case(oracle, m, n + 16, k + 16, 71, "ties")
    A, B, S, Bi = cuda(a), cuda(b), cuda(scales), cuda(bias)
    out = gemm.gemm_s8s8_requant(A[:, 1:k + 1], B[1:k + 1, 1:n + 1], S, Bi).cpu().numpy()   # misaligned bases
    assert gemm.last_kernel().startswith("generic_s8_requant")
    ref = _libs.requant_s8(oracle, _libs.ref_s8(oracle, a[:, 1:k + 1], b[1:k + 1, 1:n + 1]), scales, bias)
    assert np.array_equal(out, ref)
    # output pitch that is not a multiple of 16 bytes: byte stores on the tensor-core path
    Cbig = torch.zeros((m, n + 3), dtype=torch.int8, device="cuda")
    gemm.gemm_s8s8_requant(A[:, :96], B[:96, :n], S, Bi, out=Cbig[:, :n])
    assert gemm.last_kernel().startswith("tc_s8_requant")
    ref = _libs.requant_s8(oracle, _libs.ref_s8(oracle, a[:, :96], b[:96, :n]), scales, bias)
    assert np.array_equal(Cbig[:, :n].cpu().numpy(), ref) and (Cbig[:, n:] == 0).all()
    # K = 0: every element is requant(0) = sat(round_away(bias)); NaN / inf scales
    out = gemm.gemm_s8s8_requant(A[:, :0], B[:0, :n], S, Bi).cpu().numpy()
    assert np.array_equal(out, _libs.requant_s8(oracle, np.zeros((m, n), np.int32), scales, bias))
    weird = scales.copy()
    weird[0], weird[1], weird[2] = np.nan, np.inf, -np.inf
    out = gemm.gemm_s8s8_requant(A[:, :96], B[:96, :n], cuda(weird), None).cpu().numpy()
    assert np.array_equal(out, _libs.requant_s8(oracle, _libs.ref_s8(oracle, a[:, :96], b[:96, :n]), weird, None))
    assert (out[0] == 0).all()


def test_full_size_s8_requant_4096(gemm, oracle):
    N = 4096
    a, b, scales, bias = _rq_case(oracle, N, N, N, 81, "layer")
    A, B, S, Bi = cuda(a), cuda(b), cuda(scales), cuda(bias)
    out = gemm.gemm_s8s8_requant(A, B, S, Bi)
    assert gemm.last_kernel().startswith("tc_s8_requant_128x256")
    rows = np.arange(0, N, 31)[:128]
    ref = _libs.requant_s8(oracle, _libs.ref_s8(oracle, a[rows], b), scales[rows], bias[rows])
    assert np.array_equal(out[torch.from_numpy(rows).cuda()].cpu().numpy(), ref)
    # whole matrix against the library's own int32 product requantised on the device with torch (fp32 ops,
    # round-half-away written out): the fused epilogue and the two-pass route agree everywhere
    c32 = gemm.gemm_s8s32(A, B)
    f = c32.float() * S[:, None] + Bi[:, None]
    t = torch.trunc(f)
    t = torch.where((f - t).abs() >= 0.5, t + torch.sign(f), t).clamp(-128, 127).to(torch.int8)
    assert torch.equal(out, t)


@pytest.mark.parametrize("mode", ["x3", "x2", "f16x2"])
@pytest.mark.parametrize("m,n,k", [(300, 520, 200), (77, 96, 80), (1000, 1104, 2048), (2304, 2304, 1024)])
def test_f32_packed_b_bit_identical(gemm, oracle, m, n, k, mode):
    """b200_gemm_f32_pack_b + b200_gemm_f32_packed == b200_gemm_f32 / _acc in the same mode, bit for bit
    (same planes, same kernel), for several A against one handle (the reuse the packing interface is for)."""
    md = {"x3": gemm.F32_BF16X3, "x2": gemm.F32_BF16X2, "f16x2": gemm.F32_F16X2}[mode]
    b = _libs.gen_f32(oracle, k, n, 52)
    B = cuda(b)
    pk = gemm.PackedB(B, md)
    for seed in (51, 53):
        A = cuda(_libs.gen_f32(oracle, m, k, seed))
        ref = gemm.gemm_f32(A, B, mode=md)
        k_ref = gemm.last_kernel()
        out = gemm.gemm_f32_packed(A, pk)
        assert gemm.last_kernel() == k_ref
        assert torch.equal(out, ref)
    C0 = cuda(_libs.gen_f32(oracle, m, n, 54))
    C1, C2 = C0.clone(), C0.clone()
    gemm.gemm_f32(A, B, out=C1, mode=md, accumulate=True)
    gemm.gemm_f32_packed(A, pk, out=C2, accumulate=True)
    assert torch.equal(C1, C2)
    t = _libs.ref_f64(oracle, A.cpu().numpy(), b)
    assert rel(out.cpu().numpy(), t) <= {"x3": TOL_X3, "x2": TOL_X2, "f16x2": TOL_F16X2}[mode]
    if mode == "f16x2":
        # both operands pre-split, and a K-sliced consumer (what the row-panel plan does with B's slices):
        # A packed once, each row block of B packed as it "arrives", products accumulated into C
        pa = gemm.PackedA(A, md)
        assert torch.equal(gemm.gemm_f32_packed_ab(pa, pk, torch.empty_like(out)), out)
        if k >= 128:
            k0 = (k // 3) // 8 * 8
            Cs = torch.empty_like(out)
            for j, (a0, a1) in enumerate(((0, k0), (k0, k))):
                pbj = gemm.PackedB(B[a0:a1], md)
                gemm.gemm_f32_packed_ab(pa, pbj, Cs, a_k0=a0, accumulate=j > 0)
                pbj.close()
            assert rel(Cs.cpu().numpy(), t) <= TOL_F16X2
        pa.close()
    pk.close()


def test_f32_packed_b_errors(gemm):
    B = torch.rand(64, 48, device="cuda")
    A = torch.rand(32, 64, device="cuda")
    for md in (gemm.F32_STRICT, gemm.F32_TF32):
        with pytest.raises(gemm.B200GemmError) as e:
            gemm.PackedB(B, md)
        assert e.value.code == -3                                   # no split in these modes
    with pytest.raises(gemm.B200GemmError) as e:
        gemm.PackedA(A, gemm.F32_BF16X3)                            # A handles exist for F16X2 only
    assert e.value.code == -3
    pk = gemm.PackedB(B)                                            # AUTO = library default (F16X2)
    assert torch.equal(gemm.gemm_f32_packed(A, pk), gemm.gemm_f32(A, B, mode=gemm.F32_F16X2))
    with pytest.raises(gemm.B200GemmError) as e:
        gemm.gemm_f32_packed(torch.rand(32, 80, device="cuda"), pk)  # k does not match the handle
    assert e.value.code == -1
    assert gemm.gemm_f32_packed(torch.rand(0, 64, device="cuda"), pk).shape == (0, 48)


def test_empty_and_k_zero(gemm):
    A = torch.zeros((0, 8), device="cuda")
    B = torch.zeros((8, 5), device="cuda")
    assert gemm.gemm_f32(A, B, mode=gemm.F32_STRICT).shape == (0, 5)
    C = torch.full((6, 5), 3.0, device="cuda")
    gemm.gemm_f32(torch.zeros((6, 0), device="cuda"), torch.zeros((0, 5), device="cuda"), out=C, mode=gemm.F32_STRICT)
    assert (C == 0).all()      # C = A*B with k = 0 is the zero matrix
    Ci = torch.full((6, 5), 3, device="cuda", dtype=torch.int32)
    gemm.gemm_s8s32(torch.zeros((6, 0), device="cuda", dtype=torch.int8), torch.zeros((0, 5), device="cuda", dtype=torch.int8), out=Ci)
    assert (Ci == 0).all()


# ---- the reference's golden vectors, through the C ABI -------------------------------------------
@pytest.mark.parametrize("idx", sorted({k.split("_")[1] for k in G.files if k.startswith("f32_")}))
def test_golden_f32(gemm, idx):
    a, b = G[f"f32_{idx}_a"], G[f"f32_{idx}_b"]
    c = gemm.gemm_f32(cuda(a), cuda(b), mode=gemm.F32_STRICT).cpu().numpy()
    assert np.array_equal(c, G[f"f32_{idx}_c_naive"])                 # reference's naive REF_MMult: bit-exact
    assert np.abs(c - G[f"f32_{idx}_c_openblas"]).max() < 1e-4        # reference's OpenBLAS REF_MMult
    c = gemm.gemm_f32(cuda(a), cuda(b), mode=gemm.F32_TF32).cpu().numpy()
    assert np.abs(c - G[f"f32_{idx}_c_openblas"]).max() <= TOL_TF32 * np.abs(G[f"f32_{idx}_c_openblas"]).max()


def test_golden_ones(gemm):
    a, b, cref = G["ones_a"], G["ones_b"], G["ones_c"]
    for mode in (gemm.F32_STRICT, gemm.F32_TF32):
        assert np.array_equal(gemm.gemm_f32(cuda(a), cuda(b), mode=mode).cpu().numpy(), cref)
    assert np.array_equal(gemm.gemm_bf16(cuda(a).bfloat16(), cuda(b).bfloat16()).cpu().numpy(), cref)


@pytest.mark.parametrize("idx", sorted({k.split("_")[1] for k in G.files if k.startswith("s8_")}))
def test_golden_s8(gemm, idx):
    a, b, cref = G[f"s8_{idx}_a"], G[f"s8_{idx}_b"], G[f"s8_{idx}_c"]
    assert np.array_equal(gemm.gemm_s8s32(cuda(a), cuda(b)).cpu().numpy(), cref)
    c = np.zeros_like(cref)
    gemm.MY_MMult_int8(a.shape[0], b.shape[1], a.shape[1], a, a.shape[1], b, b.shape[1], c, b.shape[1])
    assert np.array_equal(c, cref)          # host entry = what aarch64-int8/test_MMult.c:98 calls


@pytest.mark.parametrize("mode,tol", [("strict", 0.0), ("tf32", TOL_TF32), ("x3", TOL_X3), ("x2", TOL_X2), ("f16x2", TOL_F16X2)])
@pytest.mark.parametrize("m,n,k", [(300, 520, 200), (512, 768, 1536), (77, 96, 80)])
def test_f32_accumulate_entry(gemm, oracle, m, n, k, mode, tol):
    """b200_gemm_f32_acc: C += A*B on device pointers, and K-sliced accumulation (what the multi-GPU
    row-panel pipeline does with B arriving in row chunks) equals the one-shot product."""
    md = {"strict": gemm.F32_STRICT, "tf32": gemm.F32_TF32, "x3": gemm.F32_BF16X3, "x2": gemm.F32_BF16X2,
          "f16x2": gemm.F32_F16X2}[mode]
    a, b, c0 = _libs.gen_f32(oracle, m, k, 41), _libs.gen_f32(oracle, k, n, 42), _libs.gen_f32(oracle, m, n, 43)
    A, B = cuda(a), cuda(b)
    C = cuda(c0)
    gemm.gemm_f32(A, B, out=C, mode=md, accumulate=True)
    t = _libs.ref_f64(oracle, a, b) + c0
    if mode == "strict":
        assert np.array_equal(C.cpu().numpy(), _libs.ref_f32_fma(oracle, a, b, c0))     # chain continues from C
    else:
        assert rel(C.cpu().numpy(), t) <= tol
    # K-sliced: C = A[:, :k1]*B[:k1] ; C += A[:, k1:]*B[k1:]   (strided A views, contiguous B row blocks)
    k1 = (k // 2 + 7) // 8 * 8
    C2 = torch.empty((m, n), device="cuda")
    gemm.gemm_f32(A[:, :k1], B[:k1], out=C2, mode=md)
    gemm.gemm_f32(A[:, k1:], B[k1:], out=C2, mode=md, accumulate=True)
    t2 = _libs.ref_f64(oracle, a, b)
    if mode == "strict":
        assert np.array_equal(C2.cpu().numpy(), _libs.ref_f32_fma(oracle, a, b))         # same chain, cut in two launches
    else:
        assert rel(C2.cpu().numpy(), t2) <= tol


# ---- host entry points: the CPU harness contract C += A*B ----------------------------------------
def test_host_entry_accumulates(gemm, oracle):
    m, n, k = 96, 80, 160
    a, b, c0 = _libs.gen_f32(oracle, m, k, 1), _libs.gen_f32(oracle, k, n, 2), _libs.gen_f32(oracle, m, n, 3)
    c = c0.copy()
    gemm.MY_MMult(m, n, k, a, k, b, n, c, n, mode=gemm.F32_STRICT)
    assert np.array_equal(c, _libs.ref_f32_fma(oracle, a, b, c0))
    c = c0.copy()
    gemm.MY_MMult(m, n, k, a, k, b, n, c, n, mode=gemm.F32_TF32)
    t = _libs.ref_f64(oracle, a, b) + c0
    assert rel(c, t) <= TOL_TF32


def test_host_entry_pipelined_large(gemm, oracle):
    """Above ~8 GFLOP the host entry runs a row-block pipeline over three streams (H2D / GEMM / D2H):
    same contract, and strict stays bit-exact because every row block is the same per-element chain."""
    m, n, k = 2304, 1024, 4096          # blocks of 768 -> rounded to 768? (whole pair tiles): ragged last block
    a, b, c0 = _libs.gen_f32(oracle, m, k, 51), _libs.gen_f32(oracle, k, n, 52), _libs.gen_f32(oracle, m, n, 53)
    c = c0.copy()
    gemm.MY_MMult(m, n, k, a, k, b, n, c, n, mode=gemm.F32_STRICT)
    assert np.array_equal(c, _libs.ref_f32_fma(oracle, a, b, c0))
    c = c0.copy()
    gemm.MY_MMult(m, n, k, a, k, b, n, c, n, mode=gemm.F32_BF16X3)
    assert rel(c, _libs.ref_f64(oracle, a, b) + c0) <= TOL_X3


# ---- BASELINE.json full sizes: size-independent properties ---------------------------------------
@pytest.mark.parametrize("N", [4096])
def test_full_size_properties_f32(gemm, oracle, N):
    gen = torch.Generator(device="cuda").manual_seed(5)
    A = torch.rand((N, N), device="cuda", generator=gen) * 2 - 1
    B = torch.rand((N, N), device="cuda", generator=gen) * 2 - 1
    # (1) all-ones fixture of the aarch64 harness: every element == K exactly, every mode
    ones = torch.ones((N, N), device="cuda")
    for mode in (gemm.F32_STRICT, gemm.F32_TF32):
        assert (gemm.gemm_f32(ones, ones, mode=mode) == N).all()
    # (2) row subset against the oracle: strict is bit-exact, tf32 within tolerance
    rows = torch.arange(0, N, 61, device="cuda")[:64]
    a_np, b_np = A[rows].cpu().numpy(), B.cpu().numpy()
    ref = _libs.ref_f32_fma(oracle, a_np, b_np)
    Cs = gemm.gemm_f32(A, B, mode=gemm.F32_STRICT)
    assert np.array_equal(Cs[rows].cpu().numpy(), ref)
    Ct = gemm.gemm_f32(A, B, mode=gemm.F32_TF32)
    t = _libs.ref_f64(oracle, a_np, b_np)
    assert rel(Ct[rows].cpu().numpy(), t) <= TOL_TF32
    Cx = gemm.gemm_f32(A, B, mode=gemm.F32_BF16X3)
    assert rel(Cx[rows].cpu().numpy(), t) <= TOL_X3
    # (3) whole-matrix agreement of the independent GPU paths (catches tile-scheduling holes)
    assert float((Cs - Ct).abs().max() / Cs.abs().max()) <= TOL_TF32
    assert float((Cs - Cx).abs().max() / Cs.abs().max()) <= 2 * TOL_X3
    # (4) linearity in A, exact for power-of-two scaling
    assert torch.equal(gemm.gemm_f32(A * 2, B, mode=gemm.F32_TF32), Ct * 2)
    # (5) checksum of checksums: sum_j C(i,j) == A(i,:) . rowsum(B)   (fp64 on device)
    lhs = Cs.double().sum(dim=1)
    rhs = A.double() @ B.double().sum(dim=1)
    assert float((lhs - rhs).abs().max()) <= 1e-3 * float(rhs.abs().max()) + 1e-2


@pytest.mark.parametrize("N", [4096, 8192])
def test_full_size_properties_bf16(gemm, oracle, N):
    gen = torch.Generator(device="cuda").manual_seed(6)
    A = (torch.rand((N, N), device="cuda", generator=gen) * 2 - 1).bfloat16()
    B = (torch.rand((N, N), device="cuda", generator=gen) * 2 - 1).bfloat16()
    C = gemm.gemm_bf16(A, B)
    rows = torch.arange(0, N, 127, device="cuda")[:32]
    t = _libs.ref_f64(oracle, A[rows].float().cpu().numpy(), B.float().cpu().numpy())
    assert rel(C[rows].cpu().numpy(), t) <= TOL_BF16
    ones = torch.ones((N, N), device="cuda", dtype=torch.bfloat16)
    assert (gemm.gemm_bf16(ones, ones) == N).all()
    lhs = C.double().sum(dim=1)
    rhs = A.double() @ B.double().sum(dim=1)
    assert float((lhs - rhs).abs().max()) <= 1e-4 * float(rhs.abs().max()) + 1e-2


def test_full_size_s8_4096(gemm, oracle):
    N = 4096
    a, b = _libs.gen_s8(oracle, N, N, 31), _libs.gen_s8(oracle, N, N, 32)
    A, B = cuda(a), cuda(b)
    C = gemm.gemm_s8s32(A, B)
    assert gemm.last_kernel().startswith("tc_s8")
    rows = np.arange(0, N, 29)[:128]
    assert np.array_equal(C[torch.from_numpy(rows).cuda()].cpu().numpy(), _libs.ref_s8(oracle, a[rows], b))
    # exact integer identity over the WHOLE matrix: row sums of C == A . rowsum(B) in int64
    lhs = C.long().sum(dim=1)
    rhs = (A.double() @ B.double().sum(dim=1, keepdim=True)).squeeze(1).long()   # < 2^53: exact
    assert torch.equal(lhs, rhs)
    # the reference's ramp fixture at full size (values {0,1,2})
    ar = np.zeros((N, N), np.int8)
    oracle.oracle_random_int8_ramp(N, N, _libs.P(ar), N)
    Cr = gemm.gemm_s8s32(cuda(ar), cuda(ar))
    assert np.array_equal(Cr[:64].cpu().numpy(), _libs.ref_s8(oracle, ar[:64], ar))


@pytest.mark.parametrize("mode,tol", [("strict", 2e-6), ("tf32", TOL_TF32), ("x3", TOL_X3), ("f16x2", TOL_F16X2)])
@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (1.0, 1.0), (2.5, 0.0), (-0.75, 0.5), (0.0, 2.0), (3.0, 3.0)])
@pytest.mark.parametrize("m,n,k", [(200, 136, 264), (1000, 1104, 2048), (77, 77, 77)])
def test_f32_alpha_beta(gemm, oracle, m, n, k, alpha, beta, mode, tol):
    """C = alpha*A*B + beta*C, the contract of the reference's cuBLAS comparator (cuda/MMult_cuBLAS_1.cpp:11-19:
    cublasSgemm with alpha = 1, beta = 0).  beta == 0 must not read C (NaN in C stays out of the result)."""
    md = {"strict": gemm.F32_STRICT, "tf32": gemm.F32_TF32, "x3": gemm.F32_BF16X3, "f16x2": gemm.F32_F16X2}[mode]
    a, b, c0 = _libs.gen_f32(oracle, m, k, 61), _libs.gen_f32(oracle, k, n, 62), _libs.gen_f32(oracle, m, n, 63)
    C = cuda(c0)
    if beta == 0.0:
        C[::7, ::5] = float("nan")
    gemm.gemm_f32_ex(alpha, cuda(a), cuda(b), beta, C, mode=md)
    ab = _libs.ref_f64(oracle, a, b)
    want = alpha * ab + beta * c0.astype(np.float64)
    got = C.cpu().numpy()
    assert np.isfinite(got).all()
    scale = abs(alpha) * np.abs(ab).max() + abs(beta) * np.abs(c0).max()
    assert np.abs(got - want).max() <= tol * scale + 1e-30, (gemm.last_kernel(), np.abs(got - want).max() / scale)
    if (alpha, beta) == (1.0, 0.0):
        assert torch.equal(C, gemm.gemm_f32(cuda(a), cuda(b), mode=md))
