"""Grouped bf16 and fp16 GEMMs (b200_gemm_bf16_grouped, b200_gemm_f16_grouped) and gemm(A, B, offs=offs), the shape
of torch._grouped_mm in a mixture-of-experts layer.

The rows routed to each group are stacked in one row-major A and one C; offs (int32, on the device) holds the
cumulative end rows, clamped as end_g = min(max(offs[g], end_{g-1}), total_m) with end_{-1} = 0.  Rows
[end_{g-1}, end_g) of C are computed from those rows of A and from B_g.  With the tile width forced and the split tail
off for the reference, every group must equal the single-matrix _ex call on a contiguous copy of its rows bit for bit;
the generic kernel must equal the 2-D generic call.  Output buffers start as NaN, C has padding columns, the operands
have NaN in their padding (and between the groups of B), and whole buffers are compared, so a row written to the wrong
place, a row past the last group written, or a padding element read cannot pass.

The argument checks, the schedule model, the Python refusals and the layout resolution against torch._grouped_mm on
the CPU need no GPU."""
import ctypes as C

import pytest

import test_batched_gpu as bt
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
OUT_F32, OUT_BF16, OUT_F16 = f16.OUT_F32, f16.OUT_BF16, f16.OUT_F16
KINDS16 = f16.KINDS16                 # kind: (operand dtype, C dtype, out_type, name prefix, schedule-model kind)
GROUP_LAYS = {"nn": OP_N, "nt": OP_T}  # A is always row-major
GENERIC_GRP = {"float16": "generic_f16_grp_64x64", "bfloat16": "generic_bf16_grp_64x64"}
MAX_GROUPS = 1024


# ==== model of the offsets and of the host schedule =================================================================
def clamped_ends(offs, total_m):
    """end_g = min(max(offs[g], end_{g-1}), total_m), end_{-1} = 0: the rows [end_{g-1}, end_g) of group g."""
    ends, e = [], 0
    for o in offs:
        e = min(max(int(o), e), total_m)
        ends.append(e)
    return ends


def tile_bound(total_m, groups):
    """128-row tile rows the host sizes the grid for: each group adds at most one partial tile."""
    return ts.cdiv(total_m, ts.TILE_M) + groups


def grp_pick_bn(total_m, n, groups, sms, force=0):
    """pick_bn over the tile bound (csrc/capi.cu: with_width(128, n, ..., bound))."""
    return bt.bat_pick_bn(ts.TILE_M, n, tile_bound(total_m, groups), sms, force)


def grp_schedule(total_m, n, groups, bn, sms):
    """(tiles, split, full_tiles, ctas) that b200_gemm_debug_last_schedule reports: the bound, whole tiles, the grid."""
    tiles = tile_bound(total_m, groups) * ts.cdiv(n, bn)
    return tiles, 1, tiles, min(tiles, sms)


def grp_name(kind, lay, bn):
    return f"{KINDS16[kind][3]}_grp{'' if lay == 'nn' else '_' + lay}_128x{bn}"


def test_schedule_model():
    assert clamped_ends([3, 3, 10], 12) == [3, 3, 10]
    assert clamped_ends([40, 10, -5, 300, 450, 420], 600) == [40, 40, 40, 300, 450, 450]
    assert clamped_ends([-7, 50, 5000], 300) == [0, 50, 300]
    assert tile_bound(0, 1) == 1 and tile_bound(300, 3) == 6 and tile_bound(16384, 64) == 192
    # the bound of actual tiles: sum of ceil(m_g / 128) never exceeds it, whatever the split of the rows
    for sizes in ([0, 1, 127, 128, 129, 300, 0], [1] * 64, [16384], [4000, 0, 3, 12381]):
        assert sum(ts.cdiv(s, 128) for s in sizes) <= tile_bound(sum(sizes), len(sizes))
    for sms_ in (132, 114):
        # one group of whole tiles: the single-matrix model with one extra tile row
        assert grp_pick_bn(16384, 4096, 8, sms_) == bt.bat_pick_bn(128, 4096, 128 + 8, sms_)
        for force in (128, 192, 256):
            assert grp_pick_bn(1000, 3000, 5, sms_, force) == force
        tiles, split, full, ctas = grp_schedule(300, 200, 3, 128, sms_)
        assert (tiles, split, full, ctas) == (12, 1, 12, 12)
        assert grp_schedule(16384, 14336, 8, 256, sms_) == (136 * 56, 1, 136 * 56, sms_)
    # a few groups of a small matrix fill no wave: narrow tiles
    assert grp_pick_bn(512, 512, 2, 132) == 128
    assert grp_name("bf16", "nn", 256) == "tc_bf16_grp_128x256"
    assert grp_name("f16_of16", "nt", 192) == "tc_f16_of16_grp_nt_128x192"
    assert grp_name("bf16_obf16", "nt", 128) == "tc_bf16_obf16_grp_nt_128x128"
    assert grp_name("f16", "nn", 128) == "tc_f16_grp_128x128"


# ==== argument checks (no GPU: every case returns before the device is touched) =====================================
@pytest.mark.parametrize("entry", ["bf16", "f16"])
def test_grouped_argument_validation(gemm, entry):
    lib = gemm.lib
    fn = lib.b200_gemm_bf16_grouped if entry == "bf16" else lib.b200_gemm_f16_grouped
    out16 = OUT_BF16 if entry == "bf16" else OUT_F16
    buf = (C.c_float * 4096)()
    offs = (C.c_int32 * 4)(2, 4, 6, 8)
    m, n, k, g = 8, 6, 8, 4

    def call(op_b=OP_N, mm=m, nn=n, kk=k, a=buf, lda=k, b=buf, ldb=n, sb=k * n, o=offs, groups=g, c=buf, ldc=n,
             ot=OUT_F32, alpha=0.5, beta=0.25):
        return fn(op_b, mm, nn, kk, alpha, a, lda, b, ldb, sb, o, groups, beta, c, ldc, ot, None)

    # negative sizes, groups or stride; too many groups
    for kw in ({"mm": -1}, {"nn": -1}, {"kk": -1}, {"groups": -1}, {"sb": -1}, {"groups": MAX_GROUPS + 1}):
        assert call(**kw) == -1, kw
    for kw in ({"groups": -1}, {"sb": -1}, {"groups": MAX_GROUPS + 1}, {"kk": -1}):
        assert call(mm=0, **kw) == -1, kw                    # refused even when there is nothing to do
    # bad op, ld or out_type
    for bad in (2, -1):
        assert call(op_b=bad) == -1 and call(op_b=bad, groups=0) == -1
    assert call(lda=k - 1) == -1 and call(ldb=n - 1) == -1 and call(ldc=n - 1) == -1
    assert call(op_b=OP_T, ldb=k - 1, sb=n * k) == -1
    for ot in (3, -1, 7, OUT_F16 if entry == "bf16" else OUT_BF16):
        assert call(ot=ot) == -1 and call(ot=ot, groups=0) == -1, ot
    # null pointers with work to do, offs included
    assert call(a=None) == -1 and call(b=None) == -1 and call(c=None) == -1 and call(o=None) == -1
    assert call(o=None, alpha=0.0) == -1 and call(o=None, kk=0) == -1
    # groups > 1: B_g may not overlap or be broadcast
    assert call(sb=k * n - 1) == -1 and call(sb=0) == -1
    assert call(op_b=OP_T, ldb=k, sb=n * k - 1) == -1
    assert call(ldb=n + 2, sb=k * (n + 2) - 1) == -1
    # (groups - 1) * stride_b beyond 2^60 elements
    assert call(sb=1 << 62) == -1 and call(sb=(1 << 60) // (g - 1) + 1) == -1
    # a tile bound the kernel's int work index cannot count
    big = 1 << 30
    assert call(mm=big, nn=big, lda=k, ldb=big, sb=k * big, ldc=big) == -1
    assert call(mm=(1 << 31) - 1, nn=(1 << 31) - 1, ldb=(1 << 31) - 1, sb=k * ((1 << 31) - 1),
                ldc=(1 << 31) - 1, groups=MAX_GROUPS) == -1
    # no-ops, null pointers included
    assert call(groups=0, a=None, b=None, c=None, o=None) == 0
    assert call(mm=0, a=None, b=None, c=None, o=None) == 0
    assert call(nn=0, a=None, b=None, c=None, o=None, sb=0) == 0
    assert call(groups=0, ot=out16, sb=0) == 0
    assert call(mm=0, groups=MAX_GROUPS, sb=k * n) == 0


@pytest.mark.skipif(torch is None, reason="needs torch")
def test_python_grouped_refusals(gemm):
    """Refused before any device work: the tensors here live on the CPU."""
    x = torch.zeros((10, 8), dtype=torch.bfloat16)
    w = torch.zeros((3, 8, 6), dtype=torch.bfloat16)
    offs = torch.tensor([3, 6, 10], dtype=torch.int32)
    for dt_ in (torch.float32, torch.int8):
        with pytest.raises(TypeError):
            gemm.gemm(x.to(dt_), w.to(dt_), offs=offs)
    with pytest.raises(TypeError):
        gemm.gemm(x, w.half(), offs=offs)
    bad = [dict(bias=torch.zeros(6, dtype=torch.bfloat16)), dict(activation="relu"),
           dict(offs=offs.long()), dict(offs=offs.float()), dict(offs=offs[:2]), dict(offs=offs.view(3, 1)),
           dict(offs=torch.tensor([0, 3, 0, 6, 0, 10], dtype=torch.int32)[1::2]),       # not contiguous
           dict(offs=[3, 6, 10]),                                                        # not a tensor
           dict(out=torch.zeros((6, 10)).t()),                                           # out not row-major
           dict(out=torch.zeros((10, 7))),                                               # wrong shape
           dict(out=torch.zeros((10, 6), dtype=torch.float16))]                          # wrong dtype
    for kw in bad:
        with pytest.raises(ValueError):
            gemm.gemm(x, w, **{"offs": offs, **kw})
    with pytest.raises(ValueError):
        gemm.gemm(x, w, offs=offs)                                                       # tensors on the CPU
    with pytest.raises(ValueError):
        gemm.gemm(x.t().contiguous().t(), w, offs=offs)                                  # A not row-major
    with pytest.raises(ValueError):
        gemm.gemm(x, w[0], offs=offs)                                                    # B not 3-D
    with pytest.raises(ValueError):
        gemm.gemm(x, w[:1].expand(3, 8, 6), offs=offs)                                   # broadcast B
    with pytest.raises(ValueError):
        gemm.gemm(x, torch.zeros(8 * 6 + 12, dtype=torch.bfloat16).as_strided((3, 8, 6), (6, 6, 1)), offs=offs)
    with pytest.raises(ValueError):
        gemm.gemm(x[:, :7], w, offs=offs)                                                # inner dimensions differ


@pytest.mark.skipif(torch is None, reason="needs torch")
@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_grouped_layout_matches_torch_grouped_mm(gemm, dtype):
    """On the CPU: rows [end_{g-1}, end_g) of A times B_g, with B_g read from B's storage at the (op_b, ldb, stride_b)
    that grouped_layout resolves, is what torch._grouped_mm computes, for B as stored (G, k, n), as the transposed view
    of a (G, n, k) weight, and with padded rows.  Small integers keep every product exact."""
    d = getattr(torch, dtype)
    g = torch.Generator().manual_seed(1)
    G, k, n, total_m = 4, 16, 24, 40
    x = torch.randint(-2, 3, (total_m, k), generator=g).to(d)
    offs = torch.tensor([5, 5, 23, 40], dtype=torch.int32)
    W_nk = torch.randint(-2, 3, (G, n, k), generator=g).to(d)
    W_kn = torch.randint(-2, 3, (G, k, n), generator=g).to(d)
    padded = torch.zeros((G, k + 3, n + 8), dtype=d)
    padded[:, :k, :n] = W_kn
    for B, want_op in ((W_nk.transpose(-2, -1), OP_T), (W_kn, OP_N), (padded[:, :k, :n], OP_N)):
        tm, nn, kk, op_b, ldb, sb, groups = gemm.grouped_layout(x, B, offs)
        assert (tm, nn, kk, op_b, groups) == (total_m, n, k, want_op, G)
        want = torch._grouped_mm(x, B, offs=offs)
        storage = B.as_strided((B.untyped_storage().nbytes() // B.element_size(),), (1,), 0)
        got = torch.full((total_m, n), float("nan"), dtype=d)
        lo = 0
        for gi, hi in enumerate(clamped_ends(offs.tolist(), total_m)):
            shape = (n, k) if op_b == OP_T else (k, n)
            Bg = storage.as_strided(shape, (ldb, 1), B.storage_offset() + gi * sb)
            Bg = Bg.t() if op_b == OP_T else Bg
            assert torch.equal(Bg, B[gi])
            got[lo:hi] = (x[lo:hi].double() @ Bg.double()).to(d)
            lo = hi
        assert torch.equal(got, want)


# ==== GPU helpers ===================================================================================================
def dt(name):
    return getattr(torch, name)


class Grouped:
    """One grouped problem as stored: A (total_m x k) with NaN padding, B's groups stride_b apart with NaN between them,
    offs on the device.  how: "tma" (16-element pitches), "unaligned" (A and B one element past an allocation, pitch
    cols + 1), "odd_stride" (as tma, stride_b one element longer: not a 16-byte multiple)."""

    def __init__(self, kind, sizes, n, k, op_b, seed, how="tma", trailing=0, offs=None, total_m=None):
        ind = KINDS16[kind][0]
        self.kind, self.n, self.k, self.op_b, self.how = kind, n, k, op_b, how
        self.groups = len(sizes)
        self.total_m = total_m if total_m is not None else sum(sizes) + trailing
        raw = offs if offs is not None else [sum(sizes[:i + 1]) for i in range(len(sizes))]
        self.ends = clamped_ends(raw, self.total_m)
        self.offs = torch.tensor(raw, dtype=torch.int32, device="cuda")
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.A = (torch.rand((self.total_m, k), device="cuda", generator=g) * 2 - 1).to(dt(ind))
        self.B = (torch.rand((self.groups, k, n), device="cuda", generator=g) * 2 - 1).to(dt(ind))
        off = 1 if how == "unaligned" else 0
        self.lda = k + 1 if how == "unaligned" else ts.pitch(k)
        abuf = torch.full((off + self.total_m * self.lda + 8,), float("nan"), dtype=dt(ind), device="cuda")
        self.Av = abuf.as_strided((self.total_m, k), (self.lda, 1), off)
        self.Av.copy_(self.A)
        S = self.B.transpose(1, 2) if op_b == OP_T else self.B            # groups as stored
        rows, cols = S.shape[1:]
        self.ldb = cols + 1 if how == "unaligned" else ts.pitch(cols)
        self.sb = (rows + 2) * self.ldb + (1 if how == "odd_stride" else 0)
        bbuf = torch.full((off + self.groups * self.sb + 8,), float("nan"), dtype=dt(ind), device="cuda")
        self.Bv = bbuf.as_strided((self.groups, rows, cols), (self.sb, self.ldb, 1), off)
        self.Bv.copy_(S)

    def c_buf(self, c0=None):
        """NaN-filled C (total_m x ldc, padding columns); c0 (total_m x n) in the first n columns if given."""
        buf = torch.full((self.total_m, self.n + 1 + self.n % 2), float("nan"), dtype=dt(KINDS16[self.kind][1]),
                         device="cuda")
        if c0 is not None:
            buf[:, :self.n] = c0
        return buf

    def call(self, gemm, Cb, alpha=1.0, beta=0.0, k=None):
        lib = gemm.lib
        ind, _, ot, _, _ = KINDS16[self.kind]
        fn = lib.b200_gemm_f16_grouped if ind == "float16" else lib.b200_gemm_bf16_grouped
        before = lib.b200_gemm_launch_count()
        rc = fn(self.op_b, self.total_m, self.n, self.k if k is None else k, alpha, self.Av.data_ptr(), self.lda,
                self.Bv.data_ptr(), self.ldb, self.sb, self.offs.data_ptr(), self.groups, beta, Cb.data_ptr(),
                Cb.stride(0), ot, None)
        assert rc == 0, (self.kind, rc)
        return lib.b200_gemm_launch_count() - before, gemm.last_kernel()

    def reference(self, gemm, aligned, c0=None, alpha=1.0, beta=0.0):
        """Per group, the _ex call on a contiguous copy of its rows of A and on B_g (aligned: the tensor-core kernel;
        otherwise the 2-D generic kernel), into a C of the same geometry."""
        Cr = self.c_buf(c0)
        lo = 0
        for gi, hi in enumerate(self.ends):
            if hi > lo:
                Av, lda = tr.operand(self.A[lo:hi], OP_N, aligned)
                Bv, ldb = tr.operand(self.B[gi], self.op_b, aligned)
                f16.call16(gemm, self.kind, OP_N, self.op_b, Av, lda, Bv, ldb, Cr[lo:hi], self.n, self.k, alpha, beta)
            lo = hi
        return Cr


def check(gemm, hooks, P, bn, alpha=1.0, beta=0.0, c0=None):
    """The grouped call against per-group _ex calls: route, one launch, schedule, and the whole C buffer bit for bit."""
    hooks.b200_gemm_debug_set_bn(bn)
    hooks.b200_gemm_debug_set_split_tail(0)
    Cb = P.c_buf(c0)
    launches, name = P.call(gemm, Cb, alpha, beta)
    tc = P.how == "tma"
    lay = "nt" if P.op_b == OP_T else "nn"
    want = grp_name(P.kind, lay, bn) if tc else GENERIC_GRP[KINDS16[P.kind][0]]
    assert (launches, name) == (1, want), (P.kind, lay, bn, P.how)
    if tc:
        sms_ = torch.cuda.get_device_properties(0).multi_processor_count
        assert bt.last_schedule(gemm) == grp_schedule(P.total_m, P.n, P.groups, bn, sms_)
    Cr = P.reference(gemm, tc, c0, alpha, beta)
    assert tr.same_bits(Cb, Cr), (P.kind, lay, bn, P.how, P.ends, alpha, beta)
    return Cb


# ==== bit identity with the single-matrix call ======================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_bit_identical_to_ex_every_width(gemm, hooks, kind):
    """Both B layouts, all three widths; groups of 0, 1, 127, 128, 129 and 300 rows with empty first and last groups,
    rows after the last group (NaN), and N / K tails."""
    sizes = [0, 1, 127, 128, 129, 300, 0]
    for lay, op_b in GROUP_LAYS.items():
        for bn in (256, 192, 128):
            P = Grouped(kind, sizes, bn + 8, 3 * 64 + 40, op_b, seed=bn + op_b, trailing=5)
            Cb = check(gemm, hooks, P, bn)
            assert bool(torch.isnan(Cb[P.ends[-1]:]).all())


@gpu
@pytest.mark.parametrize("kind", ["bf16", "f16_of16"])
def test_group_counts(gemm, hooks, kind):
    """G = 1, 8, 64 (random sizes, empty groups among them) and 1024 tiny groups."""
    import random
    rnd = random.Random(7)
    for lay, op_b in GROUP_LAYS.items():
        check(gemm, hooks, Grouped(kind, [200], 136, 72, op_b, 1), 128)
        check(gemm, hooks, Grouped(kind, [rnd.choice((0, 5, 130, 260)) for _ in range(8)], 200, 136, op_b, 2), 192)
        check(gemm, hooks, Grouped(kind, [rnd.choice((0, 1, 17, 129)) for _ in range(64)], 72, 64, op_b, 3), 256)
    check(gemm, hooks, Grouped(kind, [rnd.randint(0, 3) for _ in range(MAX_GROUPS)], 40, 24, OP_T, 4, trailing=9), 128)


# ==== generic route =================================================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_generic_route_bit_identical(gemm, hooks, kind):
    """Operands TMA cannot read (unaligned A and B, a stride_b that is not a 16-byte multiple) take the grouped generic
    kernel: each group as the 2-D generic call computes it."""
    sizes = [70, 0, 1, 130, 64]
    for lay, op_b in GROUP_LAYS.items():
        check(gemm, hooks, Grouped(kind, sizes, 66, 40, op_b, 5, how="unaligned", trailing=3), 128)
        check(gemm, hooks, Grouped(kind, sizes, 66, 40, op_b, 6, how="odd_stride"), 128)


# ==== alpha / beta ==================================================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
@pytest.mark.parametrize("alpha,beta", [(0.75, -1.5), (1.0, 1.0), (-2.0, 0.0)])
def test_alpha_beta_bit_identical_to_ex(gemm, hooks, kind, alpha, beta):
    """General (alpha, beta), (1, 1), and beta = 0 with NaN in C (which must not reach the result); both routes."""
    sizes = [140, 0, 70]
    total_m, n = sum(sizes) + 4, 200
    g = torch.Generator(device="cuda").manual_seed(3)
    c0 = (torch.rand((total_m, n), device="cuda", generator=g) * 2 - 1) if beta else None
    for how in ("tma", "unaligned"):
        for op_b in (OP_N, OP_T):
            P = Grouped(kind, sizes, n, 136, op_b, 8, how=how, trailing=4)
            Cb = check(gemm, hooks, P, 128, alpha, beta, c0)
            assert not bool(torch.isnan(Cb[:P.ends[-1], :n]).any())


@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_alpha_zero_and_k_zero_touch_the_grouped_rows(gemm, kind):
    """alpha = 0 or k = 0: one element-wise launch on rows [0, end_{G-1}) only, C = round_out(beta * C), NaN operands
    unread; the end is the clamped one."""
    cd = KINDS16[kind][1]
    g = torch.Generator(device="cuda").manual_seed(9)
    for offs, total_m in (([3, 0, 13, 20], 26), ([5, -3, 100], 20), ([7, 2], 15)):
        P = Grouped(kind, [1] * len(offs), 40, 24, OP_N, 1, offs=offs, total_m=total_m)
        P.Av.fill_(float("nan"))
        P.Bv.fill_(float("nan"))
        c0 = (torch.rand((total_m, 40), device="cuda", generator=g) * 4 - 2).to(dt(cd))
        end = P.ends[-1]
        for alpha, kk, beta in ((0.0, 24, 0.5), (1.0, 0, -3.0), (0.0, 24, 0.0), (2.0, 0, 0.0)):
            Cb = P.c_buf(c0)
            launches, name = P.call(gemm, Cb, alpha, beta, k=kk)
            assert (launches, name) == (1, "scale_inplace_grp" if beta else "fill_zero_grp")
            want = c0.clone()
            want[:end] = (beta * c0[:end].float()).to(c0.dtype) if beta else 0
            assert tr.same_bits(Cb[:, :40], want), (offs, alpha, kk, beta)
            assert bool(torch.isnan(Cb[:, 40:]).all())


# ==== clamped offsets ===============================================================================================
@gpu
@pytest.mark.parametrize("kind", ["bf16", "f16_of16"])
def test_clamped_offsets(gemm, hooks, kind):
    """Non-monotone, negative and too-large offsets compute the clamped groups; every other row stays NaN."""
    cases = (([40, 10, -5, 300, 450, 420], 600), ([-7, 50, 5000], 300), ([0, 0, 130], 130))
    for offs, total_m in cases:
        for how in ("tma", "unaligned"):
            P = Grouped(kind, [0] * len(offs), 72, 64, OP_T, 11, how=how, offs=offs, total_m=total_m)
            Cb = check(gemm, hooks, P, 128)
            assert bool(torch.isnan(Cb[P.ends[-1]:]).all())


# ==== CUDA graph: offsets rewritten on the device between replays ===================================================
@gpu
def test_cuda_graph_replay_with_new_offsets(gemm, hooks):
    """One captured grouped call; offs is rewritten in place between replays with three different routings (one of
    them leaving rows after the last group), and each replay matches the per-group _ex calls for the new offsets."""
    G, total_m, n, k = 8, 1000, 256, 192
    P = Grouped("bf16", [total_m // G] * G, n, k, OP_T, 21)
    hooks.b200_gemm_debug_set_bn(128)
    hooks.b200_gemm_debug_set_split_tail(0)
    A = P.Av
    B = P.Bv.transpose(1, 2)                     # (G, k, n) view of the stored (G, n, k) groups: read as op_b = T
    out = torch.full((total_m, n), float("nan"), device="cuda")
    gemm.gemm(A, B, out, offs=P.offs)            # first call: tensor maps and kernel attributes set up outside capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gemm.gemm(A, B, out, offs=P.offs)
    routings = ([125 * (i + 1) for i in range(G)],
                [600, 600, 700, 700, 900, 990, 1000, 1000],              # skewed, with empty groups
                [0, 10, 20, 30, 40, 50, 60, 900])                        # rows 900.. belong to no group
    for offs in routings:
        out.fill_(float("nan"))
        P.offs.copy_(torch.tensor(offs, dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        P.ends = clamped_ends(offs, total_m)
        ref = P.reference(gemm, True)
        assert tr.same_bits(out, ref[:, :n]), offs
        assert bool(torch.isnan(out[P.ends[-1]:]).all())


# ==== torch parity ==================================================================================================
@gpu
@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_python_moe_shapes_against_torch(gemm, sms, dtype):
    """MoE up- and down-projections: against torch._grouped_mm (where torch accepts the dtype) with a 16-bit
    tolerance, and against float64 torch.mm per group for fp32 C; the heuristic width is the model's."""
    d = dt(dtype)
    g = torch.Generator(device="cuda").manual_seed(13)
    G, dm, dff = 8, 512, 1024
    sizes = [600, 20, 0, 300, 128, 1, 700, 299]
    total_m = sum(sizes)
    offs = torch.tensor([sum(sizes[:i + 1]) for i in range(G)], dtype=torch.int32, device="cuda")
    x = ((torch.rand((total_m, dm), device="cuda", generator=g) * 2 - 1) / 8).to(d)
    W_up = ((torch.rand((G, dff, dm), device="cuda", generator=g) * 2 - 1) / 8).to(d)
    W_down = ((torch.rand((G, dm, dff), device="cuda", generator=g) * 2 - 1) / 8).to(d)
    rel16 = 2.0 ** -7 if dtype == "bfloat16" else 2.0 ** -10
    for X, W in ((x, W_up), (None, W_down)):
        if X is None:
            X = h.to(d)
        Bt = W.transpose(-2, -1)                                         # read in place: op_b = T
        h = gemm.gemm(X, Bt, offs=offs)
        bn = grp_pick_bn(total_m, Bt.shape[2], G, sms)
        assert gemm.last_kernel() == grp_name("bf16" if dtype == "bfloat16" else "f16", "nt", bn)
        assert bt.last_schedule(gemm) == grp_schedule(total_m, Bt.shape[2], G, bn, sms)
        want = torch.cat([X[lo:hi].double() @ Bt[i].double()
                          for i, (lo, hi) in enumerate(zip([0] + offs.tolist()[:-1], offs.tolist()))])
        assert float((h.double() - want).abs().max() / want.abs().max()) <= 2e-5
        y16 = gemm.gemm(X, Bt, offs=offs, out_dtype=d)
        try:
            t = torch._grouped_mm(X, Bt, offs=offs).double()
        except RuntimeError:                                             # torch has no grouped GEMM for this dtype
            t = want
        assert bool(((y16.double() - t).abs() <= 2 * rel16 * t.abs() + 2e-5 * t.abs().max()).all())
        # the (G, k, n) layout as stored, and alpha / beta into a given out
        Bn = Bt.contiguous()
        out = torch.ones((total_m, Bn.shape[2]), device="cuda")
        gemm.gemm(X, Bn, out, offs=offs, alpha=0.5, beta=-1.0)
        assert "_grp_128x" in gemm.last_kernel(), gemm.last_kernel()
        assert float((out.double() - (0.5 * want - 1.0)).abs().max() / want.abs().max()) <= 2e-5
