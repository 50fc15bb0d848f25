"""K-grouped bf16 and fp16 GEMMs (b200_gemm_bf16_grouped_k, b200_gemm_f16_grouped_k) and gemm(A, B, offs=offs) with a
2-D A and a 2-D B: torch._grouped_mm's 2-D x 2-D form, the weight gradient dW_g = dy_g^T x_g of a mixture-of-experts
layer.

offs (int32, on the device) holds cumulative ends along K, clamped as end_g = min(max(offs[g], end_{g-1}), total_k)
with end_{-1} = 0; group g contracts K rows [end_{g-1}, end_g) of op(A) (m x total_k) and op(B) (total_k x n) into a
whole C_g = C + g * stride_c.  With the tile width forced and the split tail off for the reference, every C_g must
equal the single-matrix _ex call with k = k_g on contiguous copies of its K range bit for bit (an empty group: the _ex
call with k = 0); the generic kernel must equal the 2-D generic call.  Output buffers start as NaN, the C_g have
padding columns and gaps between them, the operands have NaN in their padding and in the K rows after the last group,
and whole buffers are compared, so an element written to the wrong place, a skipped group or a K row read from the
next group (or after the last one) cannot pass.

The argument checks, the schedule model, the Python refusals and the layout resolution against torch._grouped_mm on
the CPU need no GPU."""
import ctypes as C

import pytest

import test_batched_gpu as bt
import test_f16_gemm_gpu as f16
import test_grouped_gpu as gr
import test_tile_schedules_gpu as ts
import test_transposed_ops_gpu as tr
from test_transposed_ops_gpu import hooks, sms  # noqa: F401  (fixtures: scheduling hooks reset, SM count)

try:
    import torch
except ImportError:          # the CPU tests need no torch
    torch = None

gpu = pytest.mark.gpu
OP_N, OP_T = tr.OP_N, tr.OP_T
OUT_F32, OUT_BF16, OUT_F16 = f16.OUT_F32, f16.OUT_BF16, f16.OUT_F16
KINDS16 = f16.KINDS16                 # kind: (operand dtype, C dtype, out_type, name prefix, schedule-model kind)
OPS = f16.OPS                         # layout: (op_a, op_b)
GENERIC_KGRP = {"float16": "generic_f16_kgrp_64x64", "bfloat16": "generic_bf16_kgrp_64x64"}
MAX_GROUPS = gr.MAX_GROUPS
MAX_TOTAL_K = 2 ** 31 - 65            # K row coordinates up to end + 64 stay within int32
clamped_ends = gr.clamped_ends


def _has_gpu():
    try:
        return torch is not None and torch.cuda.is_available()
    except Exception:
        return False


# ==== model of the host schedule ====================================================================================
def kg_pick_bn(m, n, groups, sms, force=0):
    """pick_bn over groups entries of m x n, as for a batch (csrc/capi.cu: with_width(m, n, ..., groups))."""
    return bt.bat_pick_bn(m, n, groups, sms, force)


def kg_schedule(m, n, groups, bn, sms):
    """(tiles, split, full_tiles, ctas) that b200_gemm_debug_last_schedule reports: every group's tiles, whole."""
    tiles = groups * ts.cdiv(m, ts.TILE_M) * ts.cdiv(n, bn)
    return tiles, 1, tiles, min(tiles, sms)


def kg_name(kind, bn):
    return f"{KINDS16[kind][3]}_kgrp_tn_128x{bn}"


def test_schedule_model():
    assert clamped_ends([5, 5, 23, 56], 56) == [5, 5, 23, 56]
    assert clamped_ends([40, 10, -5, 300, 450, 420], 400) == [40, 40, 40, 300, 400, 400]
    for sms_ in (132, 114):
        for force in (128, 192, 256):
            assert kg_pick_bn(1000, 3000, 5, sms_, force) == force
        # one group is the single-matrix model
        for m, n in ((512, 512), (4096, 4096), (200, 136)):
            assert kg_pick_bn(m, n, 1, sms_) == ts.pick_bn(m, n, sms_, "bf16")
        assert kg_schedule(200, 136, 10, 128, sms_) == (40, 1, 40, 40)
        assert kg_schedule(14336, 4096, 64, 256, sms_) == (64 * 112 * 16, 1, 64 * 112 * 16, sms_)
    # a few small groups fill no wave: narrow tiles; the MoE-sized case of this file fills several: 256
    assert kg_pick_bn(256, 256, 2, 132) == 128
    assert kg_pick_bn(2048, 1024, 8, 132) == 256
    assert kg_name("bf16", 256) == "tc_bf16_kgrp_tn_128x256"
    assert kg_name("bf16_obf16", 192) == "tc_bf16_obf16_kgrp_tn_128x192"
    assert kg_name("f16", 128) == "tc_f16_kgrp_tn_128x128"
    assert kg_name("f16_of16", 256) == "tc_f16_of16_kgrp_tn_128x256"


# ==== argument checks (no GPU: every case returns before the device is touched) =====================================
def _caller(gemm, entry):
    fn = gemm.lib.b200_gemm_bf16_grouped_k if entry == "bf16" else gemm.lib.b200_gemm_f16_grouped_k
    buf = (C.c_float * 4096)()
    offs = (C.c_int32 * 4)(2, 4, 6, 8)
    m, n, k, g = 6, 8, 8, 4

    def call(op_a=OP_T, op_b=OP_N, mm=m, nn=n, kk=k, a=buf, lda=m, b=buf, ldb=n, o=offs, groups=g, c=buf, ldc=n,
             sc=m * n, ot=OUT_F32, alpha=0.5, beta=0.25):
        return fn(op_a, op_b, mm, nn, kk, alpha, a, lda, b, ldb, o, groups, beta, c, ldc, sc, ot, None)
    return call, (m, n, k, g)


@pytest.mark.parametrize("entry", ["bf16", "f16"])
def test_grouped_k_argument_validation(gemm, entry):
    call, (m, n, k, g) = _caller(gemm, entry)
    out16 = OUT_BF16 if entry == "bf16" else OUT_F16
    # negative sizes, groups or stride; too many groups; total_k past the coordinate bound
    bad = ({"nn": -1}, {"kk": -1}, {"groups": -1}, {"sc": -1}, {"groups": MAX_GROUPS + 1}, {"kk": MAX_TOTAL_K + 1},
           {"kk": 2 ** 31 - 1})
    for kw in ({"mm": -1},) + bad:
        assert call(**kw) == -1, kw
    for kw in bad:
        assert call(mm=0, **kw) == -1, kw                    # refused even when there is nothing to do
    # the total_k bound, exactly: groups == 0 makes the call at the bound a no-op, and one past it is refused first
    assert call(groups=0, kk=MAX_TOTAL_K) == 0 and call(groups=0, kk=MAX_TOTAL_K + 1) == -1
    # bad op, ld or out_type
    for bad_op in ((2, 0), (0, 2), (-1, 0), (0, -1)):
        assert call(op_a=bad_op[0], op_b=bad_op[1]) == -1, bad_op
        assert call(op_a=bad_op[0], op_b=bad_op[1], groups=0) == -1, bad_op
    assert call(lda=m - 1) == -1 and call(ldb=n - 1) == -1 and call(ldc=n - 1) == -1
    assert call(op_a=OP_N, lda=k - 1) == -1 and call(op_b=OP_T, ldb=k - 1) == -1
    for ot in (3, -1, 7, OUT_F16 if entry == "bf16" else OUT_BF16):
        assert call(ot=ot) == -1 and call(ot=ot, groups=0) == -1, ot
    # null pointers with work to do, offs included (total_k == 0 and alpha == 0 still write every C_g)
    assert call(a=None) == -1 and call(b=None) == -1 and call(c=None) == -1 and call(o=None) == -1
    assert call(o=None, alpha=0.0) == -1 and call(o=None, kk=0) == -1 and call(c=None, kk=0) == -1
    # groups > 1: the C_g may not overlap
    assert call(sc=(m - 1) * n + n - 1) == -1 and call(sc=0) == -1
    assert call(ldc=n + 2, sc=(m - 1) * (n + 2) + n - 1) == -1
    # (groups - 1) * stride_c beyond 2^60 elements
    assert call(sc=1 << 62) == -1 and call(sc=(1 << 60) // (g - 1) + 1) == -1
    # tiles the kernel's int work index cannot count: groups * ceil(m / 128) * ceil(n / 128) > 2^30 - 1
    tm, tn = 32767, 32769                                   # tm * tn = 2^30 - 1
    big = dict(mm=128 * tm, lda=128 * tm, ldb=128 * tn + 1, ldc=128 * tn + 1, groups=1)
    assert call(nn=128 * tn + 1, **big) == -1
    assert call(mm=128 * 1024, lda=128 * 1024, nn=128 * 1024, ldb=128 * 1024, ldc=128 * 1024, sc=1 << 34,
                groups=MAX_GROUPS) == -1
    # no-ops, null pointers included
    assert call(groups=0, a=None, b=None, c=None, o=None) == 0
    assert call(mm=0, a=None, b=None, c=None, o=None) == 0
    assert call(nn=0, a=None, b=None, c=None, o=None, sc=0) == 0
    assert call(groups=0, ot=out16, sc=0) == 0
    assert call(mm=0, groups=MAX_GROUPS, sc=0) == 0


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device behaviour")
@pytest.mark.parametrize("entry", ["bf16", "f16"])
def test_grouped_k_bounds_pass_the_checks_without_device(gemm, entry):
    """The calls at the exact bounds pass every argument check and fail only for want of a device (-2)."""
    call, _ = _caller(gemm, entry)
    tm, tn = 32767, 32769
    assert call(mm=128 * tm, lda=128 * tm, nn=128 * tn, ldb=128 * tn, ldc=128 * tn, groups=1) == -2
    assert call(mm=1, lda=1, nn=1, ldb=1, ldc=1, kk=MAX_TOTAL_K, sc=1) == -2
    assert call(kk=0, a=None, b=None) == -2                 # total_k == 0 is not a no-op


@pytest.mark.skipif(torch is None, reason="needs torch")
def test_python_grouped_k_refusals(gemm):
    """Refused before any device work: the tensors here live on the CPU."""
    dy = torch.zeros((10, 6), dtype=torch.bfloat16)
    x = torch.zeros((10, 8), dtype=torch.bfloat16)
    offs = torch.tensor([3, 6, 10], dtype=torch.int32)
    for dt_ in (torch.float32, torch.int8):
        with pytest.raises(TypeError):
            gemm.gemm(dy.t().to(dt_), x.to(dt_), offs=offs)
    with pytest.raises(TypeError):
        gemm.gemm(dy.t(), x.half(), offs=offs)
    bad = [dict(bias=torch.zeros(8, dtype=torch.bfloat16)), dict(activation="relu"),
           dict(offs=offs.long()), dict(offs=offs.float()), dict(offs=offs.view(3, 1)),
           dict(offs=torch.tensor([0, 3, 0, 6, 0, 10], dtype=torch.int32)[1::2]),       # not contiguous
           dict(offs=[3, 6, 10]),                                                        # not a tensor
           dict(out=torch.zeros((3, 8, 6)).transpose(1, 2)),                             # out not row-major
           dict(out=torch.zeros((3, 6, 7))),                                             # wrong shape
           dict(out=torch.zeros((6, 8))),                                                # not one matrix per group
           dict(out=torch.zeros((6, 8)).expand(3, 6, 8)),                                # groups of out overlap
           dict(out=torch.zeros((3, 6, 8), dtype=torch.float16)),                        # wrong dtype
           dict(out_dtype=torch.float16)]
    for kw in bad:
        with pytest.raises(ValueError):
            gemm.gemm(dy.t(), x, **{"offs": offs, **kw})
    with pytest.raises(ValueError):
        gemm.gemm(dy.t(), x, offs=offs)                                                  # tensors on the CPU
    with pytest.raises(ValueError):
        gemm.gemm(dy.t(), x[:9], offs=offs)                                              # inner dimensions differ
    with pytest.raises(ValueError):
        gemm.gemm(torch.zeros((6, 20), dtype=torch.bfloat16)[:, ::2], x, offs=offs)      # A neither N nor T


def _storage_view(T, shape, ld, op):
    """The logical operand that (op, ld) reads from T's storage: op = T reads the stored transpose."""
    storage = T.as_strided((T.untyped_storage().nbytes() // T.element_size(),), (1,), 0)
    S = storage.as_strided(shape[::-1] if op == OP_T else shape, (ld, 1), T.storage_offset())
    return S.t() if op == OP_T else S


@pytest.mark.skipif(torch is None, reason="needs torch")
@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_grouped_k_layout_matches_torch_grouped_mm(gemm, dtype):
    """On the CPU: per group, op(A)[:, K_g] op(B)[K_g, :], with A and B read from their storage at the (op, ld) that
    grouped_k_layout resolves, is what torch._grouped_mm computes for every stride layout, padded rows, offsets at
    non-multiples of 64 and an empty group (zeros).  Small integers keep every product exact."""
    d = getattr(torch, dtype)
    g = torch.Generator().manual_seed(3)
    G, m, n, T = 4, 24, 40, 56
    dy = torch.randint(-2, 3, (T, m), generator=g).to(d)
    x = torch.randint(-2, 3, (T, n), generator=g).to(d)
    offs = torch.tensor([5, 5, 23, 50], dtype=torch.int32)
    dy_pad = torch.zeros((T, m + 8), dtype=d)
    dy_pad[:, :m] = dy
    x_t = x.t().contiguous()
    cases = ((dy.t(), x, OP_T, OP_N), (dy.t().contiguous(), x, OP_N, OP_N), (dy.t(), x_t.t(), OP_T, OP_T),
             (dy.t().contiguous(), x_t.t(), OP_N, OP_T), (dy_pad[:, :m].t(), x, OP_T, OP_N))
    for A, B, want_a, want_b in cases:
        mm, nn, tk, op_a, lda, op_b, ldb, groups = gemm.grouped_k_layout(A, B, offs)
        assert (mm, nn, tk, op_a, op_b, groups) == (m, n, T, want_a, want_b, G)
        Av, Bv = _storage_view(A, (m, T), lda, op_a), _storage_view(B, (T, n), ldb, op_b)
        assert torch.equal(Av, A) and torch.equal(Bv, B)
        want = torch._grouped_mm(A, B, offs=offs)
        got = torch.full((G, m, n), float("nan"), dtype=d)
        lo = 0
        for gi, hi in enumerate(clamped_ends(offs.tolist(), T)):
            got[gi] = (Av[:, lo:hi].double() @ Bv[lo:hi].double()).to(d)
            lo = hi
        assert torch.equal(got, want)
        assert not bool(got[1].any())                       # the empty group: zeros


# ==== GPU helpers ===================================================================================================
def dt(name):
    return getattr(torch, name)


def stored_nan(X, op, aligned):
    """(view passed to the library, ld): op = N stores X, op = T stores X^T, row-major, with at least one NaN padding
    column; aligned = 16-element pitch and 16-byte base (TMA-able), otherwise pitch cols + 1 and a base one element
    past an allocation."""
    S = X.t() if op == OP_T else X
    r, c = S.shape
    ld, off = (ts.pitch(c + 1), 0) if aligned else (c + 1, 1)
    buf = torch.full((off + r * ld + 8,), float("nan"), dtype=X.dtype, device="cuda")
    v = buf.as_strided((r, c), (ld, 1), off)
    v.copy_(S)
    return v, ld


class KGrouped:
    """One K-grouped problem as stored: op(A) (m x total_k) and op(B) (total_k x n) in the layout `lay`, NaN in their
    padding and in the K rows [end_{G-1}, total_k), offs on the device.  how: "tma" or "unaligned"."""

    def __init__(self, kind, sizes, m, n, lay="tn", seed=0, how="tma", trailing=0, offs=None, total_k=None):
        ind = KINDS16[kind][0]
        self.kind, self.m, self.n, self.lay, self.how = kind, m, n, lay, how
        self.op_a, self.op_b = OPS[lay]
        self.total_k = total_k if total_k is not None else sum(sizes) + trailing
        raw = offs if offs is not None else [sum(sizes[:i + 1]) for i in range(len(sizes))]
        self.groups = len(raw)
        self.ends = clamped_ends(raw, self.total_k)
        self.offs = torch.tensor(raw, dtype=torch.int32, device="cuda")
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.A = (torch.rand((m, self.total_k), device="cuda", generator=g) * 2 - 1).to(dt(ind))
        self.B = (torch.rand((self.total_k, n), device="cuda", generator=g) * 2 - 1).to(dt(ind))
        end = self.ends[-1] if self.ends else 0
        self.A[:, end:] = float("nan")                        # never read
        self.B[end:] = float("nan")
        self.restore()

    def restore(self):
        """(Re)stores A and B after the logical operands changed."""
        aligned = self.how == "tma"
        self.Av, self.lda = stored_nan(self.A, self.op_a, aligned)
        self.Bv, self.ldb = stored_nan(self.B, self.op_b, aligned)

    def c_stack(self, c0=None):
        return bt.CStack(self.kind, self.groups, self.m, self.n, c0=c0)

    def call(self, gemm, Cs, alpha=1.0, beta=0.0, total_k=None):
        lib = gemm.lib
        ind, _, ot, _, _ = KINDS16[self.kind]
        fn = lib.b200_gemm_f16_grouped_k if ind == "float16" else lib.b200_gemm_bf16_grouped_k
        before = lib.b200_gemm_launch_count()
        rc = fn(self.op_a, self.op_b, self.m, self.n, self.total_k if total_k is None else total_k, alpha,
                self.Av.data_ptr(), self.lda, self.Bv.data_ptr(), self.ldb, self.offs.data_ptr(), self.groups, beta,
                Cs.buf.data_ptr(), Cs.ldc, Cs.sc, ot, None)
        assert rc == 0, (self.kind, rc)
        return lib.b200_gemm_launch_count() - before, gemm.last_kernel()

    def reference(self, gemm, aligned, c0=None, alpha=1.0, beta=0.0):
        """Per group, the _ex call with k = k_g on contiguous copies of its K range (aligned: the tensor-core kernel;
        otherwise the 2-D generic kernel), the k == 0 call for an empty group, into a C of the same geometry."""
        Cr = self.c_stack(c0)
        lo = 0
        for gi, hi in enumerate(self.ends):
            if hi > lo:
                Av, lda = tr.operand(self.A[:, lo:hi].contiguous(), self.op_a, aligned)
                Bv, ldb = tr.operand(self.B[lo:hi].contiguous(), self.op_b, aligned)
            else:
                Av, lda, Bv, ldb = None, self.m, None, self.n
            f16.call16(gemm, self.kind, self.op_a, self.op_b, Av, lda, Bv, ldb, Cr.entry(gi), self.n, hi - lo, alpha,
                       beta)
            lo = hi
        return Cr


def check(gemm, hooks, P, bn, alpha=1.0, beta=0.0, c0=None):
    """The K-grouped call against per-group _ex calls: route, one launch, schedule, and the whole C buffer bit for bit."""
    hooks.b200_gemm_debug_set_bn(bn)
    hooks.b200_gemm_debug_set_split_tail(0)
    Cs = P.c_stack(c0)
    launches, name = P.call(gemm, Cs, alpha, beta)
    tc = P.how == "tma" and P.lay == "tn"
    want = kg_name(P.kind, bn) if tc else GENERIC_KGRP[KINDS16[P.kind][0]]
    assert (launches, name) == (1, want), (P.kind, P.lay, bn, P.how)
    if tc:
        sms_ = torch.cuda.get_device_properties(0).multi_processor_count
        assert bt.last_schedule(gemm) == kg_schedule(P.m, P.n, P.groups, bn, sms_)
    Cr = P.reference(gemm, tc, c0, alpha, beta)
    assert tr.same_bits(Cs.buf, Cr.buf), (P.kind, P.lay, bn, P.how, P.ends, alpha, beta)
    return Cs


def bits(x):
    return x.view(torch.int32 if x.element_size() == 4 else torch.int16)


SIZES = [0, 1, 15, 63, 64, 65, 127, 129, 300, 0]     # empty first and last groups; ends at non-multiples of 64


# ==== bit identity with the single-matrix call ======================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_bit_identical_to_ex_every_width(gemm, hooks, kind):
    """All three widths; groups of 0, 1, 15, 63, 64, 65, 127, 129 and 300 K rows, NaN rows after the last group, and
    M / N tails."""
    for bn in (256, 192, 128):
        check(gemm, hooks, KGrouped(kind, SIZES, 200, bn + 8, seed=bn, trailing=5), bn)
    check(gemm, hooks, KGrouped(kind, SIZES, 200, 136, seed=1, trailing=70), 128)


@gpu
@pytest.mark.parametrize("kind", ["bf16", "f16_of16"])
def test_group_counts(gemm, hooks, kind):
    """G = 1, 8 (random sizes with empty groups), 64 and 1024 tiny groups."""
    import random
    rnd = random.Random(7)
    check(gemm, hooks, KGrouped(kind, [200], 136, 72, seed=1), 128)
    check(gemm, hooks, KGrouped(kind, [rnd.choice((0, 5, 130, 260)) for _ in range(8)], 200, 136, seed=2), 192)
    check(gemm, hooks, KGrouped(kind, [rnd.choice((0, 1, 17, 129)) for _ in range(64)], 72, 64, seed=3), 256)
    check(gemm, hooks, KGrouped(kind, [rnd.randint(0, 3) for _ in range(MAX_GROUPS)], 40, 24, seed=4, trailing=9), 128)


# ==== the mask of a group's last box ================================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_next_group_inf_and_nan_never_reach_a_group(gemm, hooks, kind):
    """Group 1's K rows of A and B hold +-inf and NaN and follow group 0 (70 rows: its last box reads 58 of them);
    group 0 stays finite and bit-identical to _ex, and so does a finite group after it.  Rows after the last group
    are NaN."""
    for how in ("tma", "unaligned"):
        P = KGrouped(kind, [70, 90, 50], 136, 200, seed=5, how=how, trailing=40)
        special = torch.tensor([float("inf"), float("-inf"), float("nan")], device="cuda").to(P.A.dtype)
        P.A[:, 70:160] = special[torch.arange(P.m * 90, device="cuda") % 3].view(P.m, 90)
        P.B[70:160] = special[torch.arange(90 * P.n, device="cuda") % 3].view(90, P.n)
        P.restore()
        Cs = check(gemm, hooks, P, 128)
        for gi in (0, 2):
            assert bool(torch.isfinite(Cs.entry(gi)[:, :P.n]).all()), (how, gi)


# ==== empty groups ==================================================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_empty_groups(gemm, hooks, kind):
    """Empty groups first, in the middle, last and everywhere: with beta = 0, a NaN C and alpha = -1 they hold raw +0;
    with beta != 0, round_out(beta * C), as _ex with k = 0."""
    g = torch.Generator(device="cuda").manual_seed(6)
    for how in ("tma", "unaligned"):
        for sizes, trailing in (([0, 70, 0, 90, 0], 3), ([0, 0, 0], 50)):       # total_k == 0: see below
            P = KGrouped(kind, sizes, 136, 72, seed=7, how=how, trailing=trailing)
            Cs = check(gemm, hooks, P, 128, alpha=-1.0)
            for gi, s in enumerate(sizes):
                if s == 0:
                    assert not bool(bits(Cs.entry(gi)[:, :P.n]).any()), (how, sizes, gi)
                    assert bool(torch.isnan(Cs.entry(gi)[:, P.n:]).all())
            c0 = (torch.rand((P.groups, P.m, P.n), device="cuda", generator=g) * 4 - 2).to(dt(KINDS16[kind][1]))
            check(gemm, hooks, P, 128, alpha=-1.0, beta=-0.75, c0=c0)


# ==== clamped offsets ===============================================================================================
@gpu
@pytest.mark.parametrize("kind", ["bf16", "f16_of16"])
def test_clamped_offsets(gemm, hooks, kind):
    """Non-monotone, negative and too-large offsets contract the clamped K ranges; the groups they leave empty are
    written as empty groups."""
    cases = (([40, 10, -5, 300, 450, 420], 600), ([-7, 50, 5000], 300), ([0, 0, 130], 130))
    for offs, total_k in cases:
        for how in ("tma", "unaligned"):
            check(gemm, hooks, KGrouped(kind, [], 72, 136, seed=11, how=how, offs=offs, total_k=total_k), 128)


# ==== alpha / beta ==================================================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
@pytest.mark.parametrize("alpha,beta", [(0.75, -1.5), (1.0, 1.0), (-2.0, 0.0)])
def test_alpha_beta_bit_identical_to_ex(gemm, hooks, kind, alpha, beta):
    """General (alpha, beta), (1, 1) (gradient accumulation into C), and beta = 0 with NaN in C; both routes."""
    sizes = [140, 0, 70]
    m, n = 200, 136
    g = torch.Generator(device="cuda").manual_seed(3)
    c0 = (torch.rand((len(sizes), m, n), device="cuda", generator=g) * 2 - 1) if beta else None
    for how in ("tma", "unaligned"):
        Cs = check(gemm, hooks, KGrouped(kind, sizes, m, n, seed=8, how=how, trailing=4), 128, alpha, beta, c0)
        for gi in range(len(sizes)):
            assert not bool(torch.isnan(Cs.entry(gi)[:, :n]).any())


# ==== generic route =================================================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_generic_route_bit_identical(gemm, hooks, kind):
    """The NN, NT and TT layouts (TMA-able or not) and unaligned TN operands take the K-grouped generic kernel: each
    group as the 2-D generic call computes it on copies of its K range."""
    sizes = [70, 0, 1, 130, 64]
    for lay in ("nn", "nt", "tt"):
        check(gemm, hooks, KGrouped(kind, sizes, 66, 40, lay, seed=12, trailing=3), 128)
    for lay in ("nn", "nt", "tn", "tt"):
        check(gemm, hooks, KGrouped(kind, sizes, 66, 40, lay, seed=13, how="unaligned", trailing=3), 128)


# ==== alpha == 0 and total_k == 0 ===================================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_alpha_zero_and_total_k_zero(gemm, kind):
    """One element-wise launch over every C_g, C_g = round_out(beta * C_g) or zeros, operands (NaN) unread."""
    cd = KINDS16[kind][1]
    g = torch.Generator(device="cuda").manual_seed(9)
    P = KGrouped(kind, [3, 0, 13], 40, 24, seed=1, trailing=4)
    P.Av.fill_(float("nan"))
    P.Bv.fill_(float("nan"))
    c0 = (torch.rand((P.groups, P.m, P.n), device="cuda", generator=g) * 4 - 2).to(dt(cd))
    for alpha, tk, beta in ((0.0, P.total_k, 0.5), (1.0, 0, -3.0), (0.0, P.total_k, 0.0), (-2.0, 0, 0.0)):
        Cs = P.c_stack(c0)
        launches, name = P.call(gemm, Cs, alpha, beta, total_k=tk)
        assert (launches, name) == (1, "scale_inplace_bat" if beta else "fill_zero_bat")
        for gi in range(P.groups):
            want = (beta * c0[gi].float()).to(c0.dtype) if beta else torch.zeros_like(c0[gi])
            assert tr.same_bits(Cs.entry(gi)[:, :P.n], want), (alpha, tk, beta, gi)
            assert bool(torch.isnan(Cs.entry(gi)[:, P.n:]).all())


# ==== CUDA graph: offsets rewritten on the device between replays ===================================================
@gpu
def test_cuda_graph_replay_with_new_offsets(gemm, hooks):
    """One captured gemm(dy.t(), x, offs=offs); offs is rewritten in place between replays with three routings (one
    with empty groups, one leaving K rows after the last group), and each replay matches the per-group _ex calls."""
    G, T, m, n = 8, 1000, 192, 256
    P = KGrouped("bf16", [T // G] * G, m, n, seed=21)
    hooks.b200_gemm_debug_set_bn(128)
    hooks.b200_gemm_debug_set_split_tail(0)
    A = P.Av.t()                                  # (m, T) view of the stored (T, m) dy: read as op_a = T
    out = torch.full((G, m, n), float("nan"), device="cuda")
    gemm.gemm(A, P.Bv, out, offs=P.offs)          # first call: tensor maps and kernel attributes set up outside capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gemm.gemm(A, P.Bv, out, offs=P.offs)
    assert gemm.last_kernel() == kg_name("bf16", 128)
    routings = ([125 * (i + 1) for i in range(G)],
                [600, 600, 700, 700, 900, 990, 1000, 1000],              # skewed, with empty groups
                [0, 10, 20, 30, 40, 50, 60, 900])                        # K rows 900.. belong to no group
    for offs in routings:
        out.fill_(float("nan"))
        P.offs.copy_(torch.tensor(offs, dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        P.ends = clamped_ends(offs, T)
        ref = P.reference(gemm, True)
        for gi in range(G):
            assert tr.same_bits(out[gi], ref.entry(gi)[:, :n]), (offs, gi)


# ==== an MoE layer's training step in gemm() only ===================================================================
def zipf_sizes(T, E, empty, seed):
    """T tokens over E experts with Zipf(1) weights, expert `empty` getting none."""
    import random
    w = [0.0 if e == empty else 1.0 / (1 + (e if e < empty else e - 1)) for e in range(E)]
    rnd = random.Random(seed)
    sizes = [0] * E
    for _ in range(T):
        sizes[rnd.choices(range(E), w)[0]] += 1
    return sizes


def test_zipf_sizes():
    s = zipf_sizes(1000, 6, 2, 0)
    assert sum(s) == 1000 and s[2] == 0 and s[0] > s[1] > s[3]


@gpu
@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_python_moe_training_step_against_autograd(gemm, dtype):
    """y = x W_e^T (offs=, op_b = T), dx = dy W_e (op_b = N) and dW_e = dy_e^T x_e (the K-grouped call) of a small
    MoE layer with a Zipf routing and one empty expert, against torch autograd on float64 CPU copies: fp32 C within
    2e-5 of the largest magnitude, 16-bit C within two 16-bit ulps plus that.  The empty expert's dW is zero."""
    d = dt(dtype)
    g = torch.Generator(device="cuda").manual_seed(17)
    E, dm, dff = 6, 96, 160
    sizes = zipf_sizes(700, E, 3, 1)
    T = sum(sizes)
    offs = torch.tensor([sum(sizes[:i + 1]) for i in range(E)], dtype=torch.int32, device="cuda")
    x = ((torch.rand((T, dm), device="cuda", generator=g) * 2 - 1) / 4).to(d)
    W = ((torch.rand((E, dff, dm), device="cuda", generator=g) * 2 - 1) / 4).to(d)
    dy = ((torch.rand((T, dff), device="cuda", generator=g) * 2 - 1) / 4).to(d)
    x64 = x.double().cpu().requires_grad_()
    W64 = W.double().cpu().requires_grad_()
    bounds = [0] + offs.tolist()
    y64 = torch.cat([x64[bounds[e]:bounds[e + 1]] @ W64[e].t() for e in range(E)])
    y64.backward(dy.double().cpu())
    rel16 = 2.0 ** -7 if dtype == "bfloat16" else 2.0 ** -10
    for out_dtype in (None, d):
        r = rel16 if out_dtype is not None else 0.0
        y = gemm.gemm(x, W.transpose(-2, -1), offs=offs, out_dtype=out_dtype)
        dx = gemm.gemm(dy, W, offs=offs, out_dtype=out_dtype)
        dW = gemm.gemm(dy.t(), x, offs=offs, out_dtype=out_dtype)
        kind = {"bfloat16": "bf16", "float16": "f16"}[dtype] + ({"bfloat16": "_obf16", "float16": "_of16"}[dtype]
                                                                 if out_dtype is not None else "")
        assert gemm.last_kernel().startswith(KINDS16[kind][3] + "_kgrp_tn_"), gemm.last_kernel()
        assert tuple(dW.shape) == (E, dff, dm)
        for got, want in ((y, y64), (dx, x64.grad), (dW, W64.grad)):
            got, want = got.double().cpu(), want.detach()
            tol = 2 * r * want.abs() + 2e-5 * float(want.abs().max())
            assert bool(((got - want).abs() <= tol).all()), (out_dtype, tuple(want.shape))
        assert not bool(bits(dW[3]).any())                   # the empty expert: +0 everywhere


# ==== one MoE-sized case on the 256-wide kernel =====================================================================
@gpu
@pytest.mark.parametrize("kind", ["bf16", "f16"])
def test_moe_sized_weight_gradient(gemm, sms, kind):
    """dW_g = dy_g^T x_g for T = 8192 routed tokens, m = 2048, n = 1024, G = 8 with a Zipf routing: the heuristic takes
    the 256-wide kernel, and 16 sampled rows of every dW_g match a float64 reference within 2e-5 of their largest
    magnitude."""
    d = dt(KINDS16[kind][0])
    g = torch.Generator(device="cuda").manual_seed(23)
    T, m, n, G = 8192, 2048, 1024, 8
    sizes = zipf_sizes(T, G + 1, G, 5)[:G]
    offs = torch.tensor([sum(sizes[:i + 1]) for i in range(G)], dtype=torch.int32, device="cuda")
    dy = ((torch.rand((T, m), device="cuda", generator=g) * 2 - 1) / 8).to(d)
    x = ((torch.rand((T, n), device="cuda", generator=g) * 2 - 1) / 8).to(d)
    dW = gemm.gemm(dy.t(), x, offs=offs)
    bn = kg_pick_bn(m, n, G, sms)
    assert bn == 256 and gemm.last_kernel() == kg_name(kind, bn)
    assert bt.last_schedule(gemm) == kg_schedule(m, n, G, bn, sms)
    rows = torch.randperm(m, generator=torch.Generator().manual_seed(1))[:16].cuda()
    bounds = [0] + offs.tolist()
    for e in range(G):
        lo, hi = bounds[e], bounds[e + 1]
        want = dy[lo:hi, rows].double().t() @ x[lo:hi].double()
        err = float((dW[e, rows].double() - want).abs().max())
        assert err <= 2e-5 * max(float(want.abs().max()), 1e-30), (e, err)
