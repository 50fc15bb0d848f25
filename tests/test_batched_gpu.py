"""Strided-batched bf16 and fp16 GEMMs (b200_gemm_bf16_batched, b200_gemm_f16_batched) and the 3-D form of gemm().

Entry b of a batched call is C_b = round_out(fma(beta, float(C_b), alpha * op(A_b) op(B_b))) with X_b = X + b * stride_x.
Every route runs the whole batch in one launch.  The tensor-core kernel walks the tiles of all entries with one
persistent grid, so its tile width and its K-split tail follow from the whole batch's tile count: the schedule model
below restates that choice on top of the one in test_tile_schedules_gpu.py.  With the tile width forced and the split
tail off, every entry must equal the single-matrix _ex call on that entry bit for bit (the same tile, the same K
order); the same holds for the generic kernel against the 2-D generic call.  Output buffers start as NaN, with gaps
between the entries of C (stride_c > m * ldc) and NaN in the padding of the operands, and whole buffers are compared,
so a tile written to the wrong entry, a skipped tile or an operand row read from the next entry cannot pass.

The argument checks, the schedule model and the Python refusals need no GPU."""
import ctypes as C

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
OUT_F32, OUT_BF16, OUT_F16 = f16.OUT_F32, f16.OUT_BF16, f16.OUT_F16
LAYS = f16.LAYS
OPS = f16.OPS
KINDS16 = f16.KINDS16                 # kind: (operand dtype, C dtype, out_type, name prefix, schedule-model kind)
GENERIC_BAT = {"float16": "generic_f16_bat_64x64", "bfloat16": "generic_bf16_bat_64x64"}


# ==== schedule model ================================================================================================
def bat_pick_bn(m, n, batch, sms, force=0):
    """pick_bn over the tiles of the whole batch (csrc/capi.cu: pick_bn(..., batch))."""
    if force in (128, 192, 256):
        return force
    best, best_cost = 128, float("inf")
    for bn, eff in ((256, 1.00), (192, 0.97), (128, 0.80)):
        waves = ts.cdiv(batch * ts.cdiv(m, ts.TILE_M) * ts.cdiv(n, bn), sms)
        cost = waves * (bn / eff + 8.0)
        if cost < best_cost:
            best, best_cost = bn, cost
    return best


def bat_split(m, n, k, batch, kind, bn, sms, split_tail=True):
    """K-split parts of the last partial round of the whole batch (launch_tc); fp32 C only."""
    out_bytes = ts.KINDS[KINDS16[kind][4]].out_bytes
    rem = batch * ts.cdiv(m, ts.TILE_M) * ts.cdiv(n, bn) % sms
    if not split_tail or out_bytes != 4 or rem == 0 or rem * 8 > 1024:
        return 1
    return max(1, min(4, sms // rem, ts.cdiv(k, 64) // 8))


def bat_name(kind, lay, bn):
    return f"{KINDS16[kind][3]}_bat{'' if lay == 'nn' else '_' + lay}_128x{bn}"


def test_schedule_model_counts_the_whole_batch():
    for sms_ in (132, 114):
        # one matrix: the model is the single-matrix one
        for m, n in ((512, 512), (1000, 3000), (128, 200), (4096, 4096)):
            assert bat_pick_bn(m, n, 1, sms_) == ts.pick_bn(m, n, sms_, "bf16")
            for kind in KINDS16:
                bn = bat_pick_bn(m, n, 1, sms_)
                assert bat_split(m, n, 2048, 1, kind, bn, sms_) == ts.tc_split(m, n, 2048, KINDS16[kind][4], bn, sms_)
    # a 512 x 512 entry alone takes 128-wide tiles (16 tiles on 132 SMs); 128 entries fill many waves and take 256
    assert bat_pick_bn(512, 512, 1, 132) == 128 and bat_pick_bn(512, 512, 128, 132) == 256
    # the split tail is cut from the whole batch's last round, and only for fp32 C
    assert bat_split(128, 128, 2048, 3, "bf16", 128, 132) == 4          # 3 tiles: the only round is the tail
    assert bat_split(256, 256, 2048, 40, "f16", 128, 132) == 4          # 160 tiles: 28 in the last round
    assert bat_split(256, 256, 2048, 33, "f16", 128, 132) == 1          # 132 tiles: no partial round
    for kind in ("bf16_obf16", "f16_of16"):
        assert bat_split(128, 128, 2048, 3, kind, 128, 132) == 1
    assert bat_name("bf16", "nn", 256) == "tc_bf16_bat_128x256"
    assert bat_name("f16_of16", "nt", 128) == "tc_f16_of16_bat_nt_128x128"
    assert bat_name("bf16_obf16", "tt", 192) == "tc_bf16_obf16_bat_tt_128x192"


# ==== argument checks (no GPU: every case returns before the device is touched) =====================================
@pytest.mark.parametrize("entry", ["bf16", "f16"])
def test_batched_argument_validation(gemm, entry):
    lib = gemm.lib
    fn = lib.b200_gemm_bf16_batched if entry == "bf16" else lib.b200_gemm_f16_batched
    out16 = OUT_BF16 if entry == "bf16" else OUT_F16
    buf = (C.c_float * 4096)()
    m, n, k = 4, 6, 8

    def call(op_a=OP_N, op_b=OP_N, mm=m, nn=n, kk=k, a=buf, lda=k, sa=m * k, b=buf, ldb=n, sb=k * n, c=buf, ldc=n,
             sc=m * n, batch=3, ot=OUT_F32, alpha=0.5, beta=0.25):
        return fn(op_a, op_b, mm, nn, kk, alpha, a, lda, sa, b, ldb, sb, beta, c, ldc, sc, batch, ot, None)

    # negative batch or stride
    for kw in ({"batch": -1}, {"sa": -1}, {"sb": -16}, {"sc": -24}):
        assert call(**kw) == -1, kw
        assert call(mm=0, **kw) == -1, kw                     # refused even when there is nothing to do
    # overlapping entries of C: stride_c < (m - 1) * ldc + n
    assert call(sc=(m - 1) * n + n - 1) == -1
    assert call(ldc=n + 2, sc=(m - 1) * (n + 2) + n - 1) == -1
    assert call(sc=0) == -1
    # bad op, ld or out_type
    for bad in ((2, 0), (0, 2), (-1, 0), (0, -1)):
        assert call(op_a=bad[0], op_b=bad[1]) == -1, bad
        assert call(op_a=bad[0], op_b=bad[1], batch=0) == -1, bad
    assert call(lda=k - 1) == -1 and call(ldb=n - 1) == -1 and call(ldc=n - 1) == -1
    assert call(op_a=OP_T, lda=m - 1) == -1 and call(op_b=OP_T, ldb=k - 1) == -1
    for ot in (3, -1, 7, OUT_F16 if entry == "bf16" else OUT_BF16):
        assert call(ot=ot) == -1, ot
        assert call(ot=ot, batch=0) == -1, ot
    # null pointers with work to do
    assert call(a=None) == -1 and call(b=None) == -1 and call(c=None) == -1
    assert call(a=None, alpha=1.0, beta=0.0) == -1
    # a batch whose tiles (and split parts) the kernel's int work index cannot count
    assert call(mm=1 << 16, nn=1 << 16, batch=1 << 14, ldb=1 << 16, ldc=1 << 16, sc=1 << 32) == -1
    # absurd sizes are refused rather than wrapping 64-bit arithmetic
    big = 1 << 30
    assert call(mm=big, nn=big, kk=8, batch=big, ldb=big, ldc=big, sc=1 << 61) == -1
    assert call(sa=1 << 62) == -1 and call(sb=1 << 62) == -1 and call(sc=1 << 62) == -1
    # no-ops, null pointers included
    assert call(batch=0, a=None, b=None, c=None) == 0
    assert call(mm=0, a=None, b=None, c=None) == 0
    assert call(nn=0, a=None, b=None, c=None, sc=0) == 0
    assert call(batch=0, ot=out16, sa=0, sb=0, sc=0) == 0
    # batch == 1 is the _ex call: its own rules (here: a null A) and no stride_c rule
    assert call(batch=1, a=None) == -1
    assert call(batch=1, mm=0, sc=0) == 0


def test_batched_layout_resolution(gemm):
    lay = gemm.batched_operand_layout
    assert lay((4, 6, 10), (60, 10, 1)) == (OP_N, 10, 60)              # contiguous
    assert lay((4, 10, 6), (60, 1, 10)) == (OP_T, 10, 60)              # k.transpose(1, 2): NT
    assert lay((4, 6, 10), (0, 10, 1)) == (OP_N, 10, 0)                # expand(): broadcast
    assert lay((4, 6, 10), (0, 1, 6)) == (OP_T, 6, 0)                  # an expand()ed transposed view
    assert lay((1, 6, 10), (12345, 10, 1)) == (OP_N, 10, 0)            # size-1 batch: its stride is never used
    assert lay((4, 6, 10), (100, 16, 1)) == (OP_N, 16, 100)            # padded rows and entries
    with pytest.raises(ValueError):
        lay((4, 6, 10), (60, 20, 2))                                   # neither row-major nor transposed


@pytest.mark.skipif(torch is None, reason="needs torch")
def test_python_batched_refusals(gemm):
    """Refused before any device work: the tensors here live on the CPU."""
    a = torch.zeros((3, 4, 8), dtype=torch.bfloat16)
    b = torch.zeros((3, 8, 6), dtype=torch.bfloat16)
    for dt in (torch.float32, torch.int8):
        with pytest.raises(TypeError):
            gemm.gemm(a.to(dt), b.to(dt))
    with pytest.raises(TypeError):
        gemm.gemm(a, b.half())
    with pytest.raises(ValueError):
        gemm.gemm(a, b, bias=torch.zeros(6, dtype=torch.bfloat16))
    with pytest.raises(ValueError):
        gemm.gemm(a, b, activation="relu")
    with pytest.raises(ValueError):
        gemm.gemm(a, torch.zeros((2, 8, 6), dtype=torch.bfloat16))          # unequal batch sizes
    with pytest.raises(ValueError):
        gemm.gemm(a, b[0])                                                   # 3-D against 2-D: pass an expand()ed view
    with pytest.raises(ValueError):
        gemm.gemm(a, b, out=torch.zeros((3, 6, 4)).transpose(1, 2))          # out not row-major
    with pytest.raises(ValueError):
        gemm.gemm(a, b, out=torch.zeros((3, 4, 7)))                          # wrong shape


# ==== GPU helpers ===================================================================================================
def dt(name):
    return getattr(torch, name)


def logical(kind, batch, m, n, k, seed, dyadic=False):
    """A (batch x m x k) and B (batch x k x n) of the kind's operand type."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if dyadic:
        A = torch.randint(-8, 9, (batch, m, k), device="cuda", generator=g).float() / 8
        B = torch.randint(-8, 9, (batch, k, n), device="cuda", generator=g).float() / 8
    else:
        A = torch.rand((batch, m, k), device="cuda", generator=g) * 2 - 1
        B = torch.rand((batch, k, n), device="cuda", generator=g) * 2 - 1
    d = dt(KINDS16[kind][0])
    return A.to(d), B.to(d)


class Stack:
    """One operand of a batch as stored for op: entry b at base + b * stride (elements), NaN in every padding element.
    how: "tma" (16-element ld, entries gap_rows apart), "unaligned" (base one element past the allocation, ld cols + 1),
    "odd_stride" (as tma, stride one element longer: not a 16-byte multiple), "overlap" (stride = ld: entries share rows),
    "bcast" (stride 0: entry 0 for every b)."""

    def __init__(self, X3, op, how="tma", gap_rows=3):
        S = X3.transpose(1, 2) if op == OP_T else X3
        nb, r, c = S.shape
        self.op, self.rows, self.cols, self.how = op, r, c, how
        self.ld = c + 1 if how == "unaligned" else ts.pitch(c)
        off = 1 if how == "unaligned" else 0
        if how == "bcast":
            self.stride = 0
        elif how == "overlap":
            self.stride = self.ld
        else:
            self.stride = (r + gap_rows) * self.ld + (1 if how == "odd_stride" else 0)
        size = off + max(nb - 1, 0) * self.stride + r * self.ld + 8
        self.buf = torch.full((size,), float("nan"), dtype=S.dtype, device="cuda")
        self.off = off
        if how == "overlap":              # the entries are windows of one random buffer: their values are what they read
            g = torch.Generator(device="cuda").manual_seed(nb * 1000 + r)
            self.buf.copy_((torch.rand(size, device="cuda", generator=g) * 2 - 1).to(S.dtype))
        elif how == "bcast":
            self.entry(0).copy_(S[0])
        elif nb:
            self.buf.as_strided((nb, r, c), (self.stride, self.ld, 1), off).copy_(S)

    def entry(self, b):
        """Entry b as stored (rows x cols view of the buffer)."""
        return self.buf.as_strided((self.rows, self.cols), (self.ld, 1), self.off + b * self.stride)

    def ptr(self, b=0):
        return self.buf.data_ptr() + (self.off + b * self.stride) * self.buf.element_size()


class CStack:
    """C of a batch: entries stride_c = m * ldc + gap apart (gap > 0), NaN everywhere first; c0 (batch x m x n) into
    the entries if given."""

    def __init__(self, kind, batch, m, n, ldc=None, gap=5, c0=None):
        self.ldc = ldc or n + 1 + n % 2
        self.m, self.n, self.batch = m, n, batch
        self.sc = m * self.ldc + gap
        self.buf = torch.full((max(batch - 1, 0) * self.sc + m * self.ldc + gap,), float("nan"),
                              dtype=dt(KINDS16[kind][1]), device="cuda")
        if c0 is not None:
            for b in range(batch):
                self.entry(b)[:, :n] = c0[b]

    def entry(self, b):
        return self.buf.as_strided((self.m, self.ldc), (self.ldc, 1), b * self.sc)


def last_schedule(gemm):
    """(tiles, split, full_tiles, ctas) of the library's last tensor-core launch (b200_gemm_debug_last_schedule)."""
    v = [C.c_int(-1) for _ in range(4)]
    gemm.lib.b200_gemm_debug_last_schedule(*[C.byref(x) for x in v])
    return tuple(x.value for x in v)


def want_schedule(m, n, k, batch, kind, bn, sms, split_tail=True):
    """The schedule model's (tiles, split, full_tiles, ctas) for a batched tensor-core call."""
    tiles = batch * ts.cdiv(m, ts.TILE_M) * ts.cdiv(n, bn)
    split = bat_split(m, n, k, batch, kind, bn, sms, split_tail)
    full = tiles - tiles % sms if split > 1 else tiles
    return tiles, split, full, min(full + (tiles - full) * split, sms)


def call_batched(gemm, kind, op_a, op_b, m, n, k, SA, SB, Cs, batch, alpha=1.0, beta=0.0):
    """One batched call; returns (launches issued, kernel name)."""
    lib = gemm.lib
    ind, _, ot, _, _ = KINDS16[kind]
    fn = lib.b200_gemm_f16_batched if ind == "float16" else lib.b200_gemm_bf16_batched
    before = lib.b200_gemm_launch_count()
    rc = fn(op_a, op_b, m, n, k, alpha, SA.ptr(), SA.ld, SA.stride, SB.ptr(), SB.ld, SB.stride, beta, Cs.buf.data_ptr(),
            Cs.ldc, Cs.sc, batch, ot, None)
    assert rc == 0, (kind, rc)
    return lib.b200_gemm_launch_count() - before, gemm.last_kernel()


def reference(gemm, kind, op_a, op_b, m, n, k, SA, SB, batch, aligned, alpha=1.0, beta=0.0, c0=None, gap=5, ldc=None):
    """The same batch as `batch` single-matrix _ex calls, each on copies of one entry's operands stored aligned (the
    tensor-core kernel) or not (the generic kernel), into a C of the batched call's geometry."""
    Cr = CStack(kind, batch, m, n, ldc=ldc, gap=gap, c0=c0)
    for b in range(batch):
        Av, lda = tr.operand(_logical_of(SA, b, op_a, m, k), op_a, aligned)
        Bv, ldb = tr.operand(_logical_of(SB, b, op_b, k, n), op_b, aligned)
        f16.call16(gemm, kind, op_a, op_b, Av, lda, Bv, ldb, Cr.entry(b), n, k, alpha, beta)
    return Cr


def _logical_of(S, b, op, rows, cols):
    """Logical rows x cols operand of entry b (entry 0 for a broadcast operand)."""
    e = S.entry(0 if S.stride == 0 else b)
    assert tuple(e.shape) == ((cols, rows) if op == OP_T else (rows, cols))
    return (e.t() if op == OP_T else e).contiguous()


def same_bits(x, y):
    return tr.same_bits(x, y)


def check_case(gemm, hooks, kind, lay, m, n, k, batch, bn, how_a="tma", how_b="tma", alpha=1.0, beta=0.0, seed=1,
               c0=None, ldc=None, gap=5):
    """The batched call against per-entry _ex calls: route, one launch, and the whole C buffer bit for bit."""
    op_a, op_b = OPS[lay]
    A, B = logical(kind, batch, m, n, k, seed)
    SA, SB = Stack(A, op_a, how_a), Stack(B, op_b, how_b)
    hooks.b200_gemm_debug_set_bn(bn)
    hooks.b200_gemm_debug_set_split_tail(0)
    Cs = CStack(kind, batch, m, n, ldc=ldc, gap=gap, c0=c0)
    launches, name = call_batched(gemm, kind, op_a, op_b, m, n, k, SA, SB, Cs, batch, alpha, beta)
    tc = all(h in ("tma", "bcast") for h in (how_a, how_b))
    want = bat_name(kind, lay, bn) if tc else GENERIC_BAT[KINDS16[kind][0]]
    assert (launches, name) == (1, want), (kind, lay, m, n, k, batch, bn, how_a, how_b)
    if tc:                                  # one grid over every entry's tiles, whole tiles only
        sms_ = torch.cuda.get_device_properties(0).multi_processor_count
        assert last_schedule(gemm) == want_schedule(m, n, k, batch, kind, bn, sms_, split_tail=False)
    Cr = reference(gemm, kind, op_a, op_b, m, n, k, SA, SB, batch, tc, alpha, beta, c0, gap=gap, ldc=ldc)
    assert same_bits(Cs.buf, Cr.buf), (kind, lay, m, n, k, batch, bn, how_a, how_b, alpha, beta)
    return Cs


# ==== bit identity with the single-matrix call ======================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_bit_identical_to_ex_every_layout_and_width(gemm, hooks, kind):
    """Both kinds, both C types, all four layouts, all three widths, M / N / K tails, batch 3 and 2."""
    for lay in LAYS:
        for bn in (256, 192, 128):
            for i, (m, n, k, batch) in enumerate(((129, bn + 8, 3 * 64 + 40, 3), (1, 2 * bn - 8, 72, 2))):
                check_case(gemm, hooks, kind, lay, m, n, k, batch, bn, seed=i + 10 * bn)


@gpu
@pytest.mark.parametrize("kind", ["bf16", "f16_of16"])
def test_bit_identical_batch_sizes(gemm, hooks, sms, kind):
    """batch 7, and more than two SMs' worth of tiles (1 tile per entry), every layout."""
    for lay in LAYS:
        check_case(gemm, hooks, kind, lay, 200, 136, 264, 7, 128)
        check_case(gemm, hooks, kind, lay, 100, 120, 72, 2 * sms + 5, 128)


@gpu
@pytest.mark.parametrize("kind", ["bf16", "f16", "bf16_obf16"])
def test_broadcast_and_padded_strides(gemm, hooks, kind):
    """stride_a = 0 and stride_b = 0 (one operand for every entry), padded entries, and C with a 16-byte-aligned entry
    stride (vector stores) as well as an odd one."""
    for lay in LAYS:
        check_case(gemm, hooks, kind, lay, 130, 72, 136, 3, 128, how_a="bcast")
        check_case(gemm, hooks, kind, lay, 130, 72, 136, 3, 192, how_b="bcast")
        check_case(gemm, hooks, kind, lay, 130, 200, 100, 4, 256, ldc=ts.pitch(200), gap=16)


# ==== split tail (fp32 C): dyadic known answers =====================================================================
@gpu
@pytest.mark.parametrize("kind", ["bf16", "f16"])
def test_split_tail_known_answer(gemm, hooks, sms, kind):
    """With the split tail on, K parts of the whole batch's last round are folded in order; dyadic operands make every
    partial sum exact, so C must be the exact product bit for bit (also with beta * C folded by part 0).  The schedule
    the library took is read back: the split is cut from the whole batch's tile count, not per entry."""
    k = 2048 + 64 * 5 + 24                                               # 37 k-blocks: uneven parts
    rounds = (128, 128, 3), (256, 256, sms // 4 + 7)                     # only round is the tail / a partial last round
    for lay in ("nn", "nt", "tn"):
        op_a, op_b = OPS[lay]
        for m, n, batch in rounds:
            split = bat_split(m, n, k, batch, kind, 128, sms)
            assert split > 1, (m, n, batch, split)
            A, B = logical(kind, batch, m, n, k, 5, dyadic=True)
            SA, SB = Stack(A, op_a), Stack(B, op_b)
            hooks.b200_gemm_debug_set_bn(128)
            c0 = torch.randint(-8, 9, (batch, m, n), device="cuda").float() / 4
            for alpha, beta in ((1.0, 0.0), (2.0, 0.5)):
                Cs = CStack(kind, batch, m, n, c0=c0 if beta else None)
                launches, name = call_batched(gemm, kind, op_a, op_b, m, n, k, SA, SB, Cs, batch, alpha, beta)
                assert (launches, name) == (1, bat_name(kind, lay, 128))
                got = last_schedule(gemm)
                assert got == want_schedule(m, n, k, batch, kind, 128, sms), (lay, m, n, batch, got)
                assert got[1] == split and got[2] < got[0]
                want = alpha * (A.double() @ B.double()) + (beta * c0.double() if beta else 0)
                for b in range(batch):
                    e = Cs.entry(b)
                    assert torch.equal(e[:, :n], want[b].float()), (lay, m, n, batch, b, alpha, beta)
                    assert bool(torch.isnan(e[:, n:]).all())
                gaps = torch.ones_like(Cs.buf, dtype=torch.bool)
                for b in range(batch):
                    gaps[b * Cs.sc: b * Cs.sc + m * Cs.ldc].view(m, Cs.ldc)[:, :n] = False
                assert bool(torch.isnan(Cs.buf[gaps]).all())


# ==== alpha / beta ==================================================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
@pytest.mark.parametrize("alpha,beta", [(0.75, -1.5), (1.0, 1.0), (-2.0, 0.0)])
def test_alpha_beta_bit_identical_to_ex(gemm, hooks, kind, alpha, beta):
    """General (alpha, beta), (1, 1), and beta = 0 with NaN in C (which must not reach the result)."""
    batch, m, n = 3, 140, 200
    g = torch.Generator(device="cuda").manual_seed(3)
    c0 = (torch.rand((batch, m, n), device="cuda", generator=g) * 2 - 1) if beta else None
    for lay in ("nn", "tt"):
        Cs = check_case(gemm, hooks, kind, lay, m, n, 136, batch, 128, alpha=alpha, beta=beta, c0=c0)
        for b in range(batch):
            assert not bool(torch.isnan(Cs.entry(b)[:, :n]).any())
        check_case(gemm, hooks, kind, lay, m, n, 136, batch, 128, how_a="unaligned", alpha=alpha, beta=beta, c0=c0)


@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_alpha_zero_and_k_zero_never_read_operands(gemm, kind):
    """alpha = 0 or k = 0: one element-wise launch over every entry, C = round_out(beta * C), NaN operands unread."""
    batch, m, n, k = 5, 33, 40, 24
    ind = KINDS16[kind][0]
    SA = Stack(torch.full((batch, m, k), float("nan"), dtype=dt(ind), device="cuda"), OP_N)
    SB = Stack(torch.full((batch, k, n), float("nan"), dtype=dt(ind), device="cuda"), OP_N)
    g = torch.Generator(device="cuda").manual_seed(9)
    c0 = (torch.rand((batch, m, n), device="cuda", generator=g) * 4 - 2).to(dt(KINDS16[kind][1]))
    for alpha, kk, beta in ((0.0, k, 0.5), (1.0, 0, -3.0), (0.0, k, 0.0), (2.0, 0, 0.0)):
        Cs = CStack(kind, batch, m, n, c0=c0)
        launches, name = call_batched(gemm, kind, OP_N, OP_N, m, n, kk, SA, SB, Cs, batch, alpha, beta)
        assert (launches, name) == (1, "scale_inplace_bat" if beta else "fill_zero_bat")
        want = (beta * c0.float()).to(c0.dtype) if beta else torch.zeros_like(c0)
        for b in range(batch):
            assert tr.same_bits(Cs.entry(b)[:, :n], want[b]), (alpha, kk, beta, b)
            assert bool(torch.isnan(Cs.entry(b)[:, n:]).all())


# ==== generic route =================================================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_generic_route_bit_identical(gemm, hooks, kind):
    """Operands TMA cannot read (unaligned base, an entry stride that is not a 16-byte multiple) and overlapping input
    entries (0 < stride < rows x ld) take the batched generic kernel: each entry as the 2-D generic call computes it."""
    for lay in LAYS:
        check_case(gemm, hooks, kind, lay, 70, 66, 40, 3, 128, how_a="unaligned", how_b="unaligned")
        check_case(gemm, hooks, kind, lay, 70, 66, 40, 3, 128, how_b="odd_stride")
    check_case(gemm, hooks, kind, "nn", 70, 66, 40, 3, 128, how_a="overlap")
    check_case(gemm, hooks, kind, "nt", 70, 66, 40, 3, 128, how_b="overlap")


@gpu
def test_generic_route_batch_above_grid_z(gemm, hooks):
    """More entries than gridDim.z allows (65 535): the kernel loops over the rest."""
    kind, batch, m, n, k = "bf16", 65535 + 70, 3, 5, 7
    A, B = logical(kind, batch, m, n, k, 4)
    SA, SB = Stack(A, OP_N, "unaligned", 0), Stack(B, OP_N, "unaligned", 0)
    Cs = CStack(kind, batch, m, n, gap=1)
    launches, name = call_batched(gemm, kind, OP_N, OP_N, m, n, k, SA, SB, Cs, batch)
    assert (launches, name) == (1, GENERIC_BAT["bfloat16"])
    want = A.float() @ B.float()            # the generic kernel accumulates in k order with fmaf; compare a sample too
    got = torch.stack([Cs.entry(b)[:, :n] for b in (0, 1, 65534, 65535, batch - 1)])
    assert torch.allclose(got, want[[0, 1, 65534, 65535, batch - 1]], rtol=1e-5, atol=1e-5)
    for b in (0, 65535, batch - 1):         # bit for bit against the 2-D generic call on that entry
        Av, lda = tr.operand(A[b], OP_N, False)
        Bv, ldb = tr.operand(B[b], OP_N, False)
        ref = f16.out_buf16(kind, m, n)
        f16.call16(gemm, kind, OP_N, OP_N, Av, lda, Bv, ldb, ref, n, k)
        assert same_bits(Cs.entry(b)[:, :n], ref[:, :n]), b
    assert bool(torch.isnan(Cs.buf.view(-1)[m * Cs.ldc::Cs.sc]).all())      # the gap element after every entry


# ==== batch == 1 ====================================================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS16))
def test_batch_one_is_the_ex_call(gemm, hooks, kind):
    m, n, k = 300, 260, 200
    for lay in ("nn", "nt"):
        op_a, op_b = OPS[lay]
        for aligned in (True, False):
            A, B = logical(kind, 1, m, n, k, 6)
            SA, SB = Stack(A, op_a, "tma" if aligned else "unaligned"), Stack(B, op_b, "tma" if aligned else "unaligned")
            Cs = CStack(kind, 1, m, n)
            got = call_batched(gemm, kind, op_a, op_b, m, n, k, SA, SB, Cs, 1, 0.5, 0.0)
            ref = f16.out_buf16(kind, m, n)
            lib = gemm.lib
            fn = lib.b200_gemm_f16_ex if KINDS16[kind][0] == "float16" else lib.b200_gemm_bf16_ex
            before = lib.b200_gemm_launch_count()
            assert fn(op_a, op_b, m, n, k, 0.5, SA.ptr(), SA.ld, SB.ptr(), SB.ld, 0.0, ref.data_ptr(), ref.stride(0),
                      KINDS16[kind][2], None) == 0
            assert got == (lib.b200_gemm_launch_count() - before, gemm.last_kernel())
            assert "_bat" not in got[1]
            assert same_bits(Cs.entry(0)[:, :n], ref[:, :n])


# ==== model-predicted widths and names ==============================================================================
@gpu
@pytest.mark.parametrize("kind", ["bf16", "f16_of16"])
def test_heuristic_width_from_the_whole_batch(gemm, hooks, sms, kind):
    """Without a forced width the kernel name is the one the model picks for the whole batch."""
    for m, n, k, batch in ((512, 512, 64, 1), (512, 512, 64, 128), (256, 1000, 72, 9)):
        A, B = logical(kind, batch, m, n, k, 8)
        SA, SB = Stack(A, OP_N), Stack(B, OP_T)
        Cs = CStack(kind, batch, m, n)
        launches, name = call_batched(gemm, kind, OP_N, OP_T, m, n, k, SA, SB, Cs, batch)
        bn = bat_pick_bn(m, n, batch, sms)
        want = bat_name(kind, "nt", bn) if batch > 1 else f"{KINDS16[kind][3]}_nt_128x{bn}"
        assert (launches, name) == (1, want), (m, n, batch)
        assert last_schedule(gemm) == want_schedule(m, n, k, batch, kind, bn, sms), (m, n, batch)


# ==== Python ========================================================================================================
@gpu
@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_python_attention_shapes_against_bmm(gemm, dtype):
    d = dt(dtype)
    g = torch.Generator(device="cuda").manual_seed(11)
    bh, s, hd = 6, 200, 64
    q = (torch.rand((bh, s, hd), device="cuda", generator=g) * 2 - 1).to(d)
    kk = (torch.rand((bh, s, hd), device="cuda", generator=g) * 2 - 1).to(d)
    v = (torch.rand((bh, s, hd), device="cuda", generator=g) * 2 - 1).to(d)
    rel16 = 2.0 ** -7 if dtype == "bfloat16" else 2.0 ** -10
    # q @ k^T: k.transpose(1, 2) is read in place (NT kernel, no copy)
    s32 = gemm.gemm(q, kk.transpose(1, 2))
    assert gemm.last_kernel().startswith(("tc_bf16_bat_nt_", "tc_f16_bat_nt_")), gemm.last_kernel()
    t = q.double() @ kk.double().transpose(1, 2)
    assert float((s32.double() - t).abs().max() / t.abs().max()) <= 2e-5
    s16 = gemm.gemm(q, kk.transpose(1, 2), out_dtype=d)
    tb = torch.bmm(q, kk.transpose(1, 2)).double()
    assert bool(((s16.double() - tb).abs() <= rel16 * tb.abs() + 2e-5 * tb.abs().max()).all())
    # p @ v (NN)
    p = s16.softmax(-1)
    o = gemm.gemm(p, v, out_dtype=d)
    assert "_bat_128x" in gemm.last_kernel(), gemm.last_kernel()
    tb = torch.bmm(p, v).double()
    assert bool(((o.double() - tb).abs() <= rel16 * tb.abs() + 2e-5 * tb.abs().max()).all())
    # an expand()ed operand (stride 0) is read in place
    w = (torch.rand((hd, 96), device="cuda", generator=g) * 2 - 1).to(d)
    y = gemm.gemm(q, w.unsqueeze(0).expand(bh, hd, 96))
    t = q.double() @ w.double()
    assert float((y.double() - t).abs().max() / t.abs().max()) <= 2e-5


@gpu
@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_python_baddbmm_alpha_beta(gemm, dtype):
    d = dt(dtype)
    g = torch.Generator(device="cuda").manual_seed(12)
    a = (torch.rand((4, 130, 72), device="cuda", generator=g) * 2 - 1).to(d)
    b = (torch.rand((4, 72, 90), device="cuda", generator=g) * 2 - 1).to(d)
    c = torch.rand((4, 130, 90), device="cuda", generator=g) * 2 - 1
    out = c.clone()
    gemm.gemm(a, b, out=out, alpha=0.5, beta=-2.0)
    t = torch.baddbmm(c.double(), a.double(), b.double(), beta=-2.0, alpha=0.5)
    assert float((out.double() - t).abs().max() / t.abs().max()) <= 2e-5
    one = gemm.gemm(a[:1], b[:1])                      # a batch of one is the 2-D call
    assert "_bat" not in gemm.last_kernel()
    assert torch.equal(one[0], gemm.gemm(a[0], b[0]))
