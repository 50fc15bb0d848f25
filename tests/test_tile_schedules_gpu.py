"""Every tile schedule of the wgmma and FFMA kernels against plain high-precision references.

The persistent tensor-core kernel picks one of three tile widths, walks the tiles in raster groups of
tile rows and cuts the last partial round of tiles along K (the split tail: 2-4 parts computed by
different CTAs and folded into C in order).  The strict fp32 kernels (128x128 and the 128x256 "fat"
kernel) issue the last round as half tiles.  Which of these paths a shape takes depends on the SM
count, so the shapes are generated from a Python restatement of the host-side choices (the schedule
model below, read with the device's SM count), and every case asserts that the model gives the path it
is meant to cover.  The model tests at the top need no GPU.

References: torch float64 matmul on the device (an implementation independent of this library, exact
for int8 because every partial sum stays below 2^53) and the CPU oracle for the bit-exact strict path.
Every output buffer starts as NaN (or a sentinel) so that a tile the schedule skips cannot pass, and
the whole matrix is compared.  The scheduling hooks are process-global: the `hooks` fixture puts the
defaults back after every test, whether it passed or not."""
import math

import numpy as np
import pytest

import _libs

try:
    import torch
except ImportError:          # the model tests below need no torch
    torch = None

gpu = pytest.mark.gpu

# tolerances of test_gpu_parity.py (normwise: max |C - Cref| / max |Cref|)
TOL = {"bf16": 2e-5, "tf32": 1e-3, "bf16x3": 1e-5, "bf16x2": 4e-5, "f16x2": 1e-5}
TOL_STRICT = 2e-6            # strict / generic fp32 under a general alpha, beta (test_f32_alpha_beta)


# ==== schedule model ====================================================================================
# A restatement of the host-side tile schedule of csrc/capi.cu:
#   pick_bn            -> pick_bn()                  (tile width heuristic, b200_gemm_debug_set_bn override)
#   launch_tc          -> tc_split(), group_m()      (split of the last partial round: rem = tiles % sms,
#                                                     split = min(4, sms // rem, num_kb // 8), 1 when
#                                                     rem * 8 epilogue warps exceed a 1024-int flag slot;
#                                                     group_m = group rows / 128, default 2048 rows)
#   launch_ffma        -> ffma_halves()              (half tiles when the last round is at most half full)
#   strict_tma         -> ffma_fat()                 (the fat kernel from 96 of its 128x256 tiles)
# BK is one 128-byte swizzled row of K per stage (64-byte rows for the split fp32 modes), TcConfig in
# csrc/gemm_tc.cuh.  If a heuristic there changes, update it here: the generators below then still aim
# at every path, and the model assertions of each GPU case fail instead of quietly losing coverage.
class Kind:
    def __init__(self, bk, out_bytes, widths, name):
        self.bk, self.out_bytes, self.widths, self.name = bk, out_bytes, widths, name


KINDS = {
    "bf16": Kind(64, 4, (128, 192, 256), "tc_bf16"),              # bf16 in, fp32 out
    "bf16_obf16": Kind(64, 2, (128, 192, 256), "tc_bf16_obf16"),  # bf16 in, bf16 out
    "tf32": Kind(32, 4, (128, 192, 256), "tc_tf32"),
    "s8": Kind(128, 4, (128, 256), "tc_s8"),                      # int8 in, int32 out
    "s8_requant": Kind(128, 1, (128, 256), "tc_s8_requant"),      # int8 in, int8 out
    "bf16x3": Kind(32, 4, (128,), "tc_bf16x3"),
    "bf16x2": Kind(32, 4, (128,), "tc_bf16x2"),
    "f16x2": Kind(32, 4, (128,), "tc_f16x2"),
}
SPLIT_KINDS = ("bf16", "tf32", "s8", "bf16x3", "bf16x2", "f16x2")     # fp32 / int32 out: the split tail applies
F32_KINDS = ("tf32", "bf16x3", "bf16x2", "f16x2")                     # b200_gemm_f32 modes (accumulate, alpha/beta)
TILE_M = 128


def cdiv(a, b):
    return -(-a // b)


def pick_bn(m, n, sms, kind, force=0):
    widths = KINDS[kind].widths
    if len(widths) == 1:
        return widths[0]
    if force in widths:
        return force
    best, best_cost = 128, math.inf
    for bn, eff in ((256, 1.00), (192, 0.97), (128, 0.80)):
        if bn not in widths:
            continue
        waves = cdiv(cdiv(m, TILE_M) * cdiv(n, bn), sms)
        cost = waves * (bn / eff + 8.0)
        if cost < best_cost:
            best, best_cost = bn, cost
    return best


def tc_split(m, n, k, kind, bn, sms, split_tail=True):
    kd = KINDS[kind]
    rem = cdiv(m, TILE_M) * cdiv(n, bn) % sms
    if not split_tail or kd.out_bytes != 4 or rem == 0:
        return 1
    if rem * 8 > 1024:
        return 1
    return max(1, min(4, sms // rem, cdiv(k, kd.bk) // 8))


def split_parts(num_kb, split):
    """k-block ranges of the parts of one split tile (work_item in csrc/gemm_tc.cuh)."""
    return [(num_kb * p // split, num_kb * (p + 1) // split) for p in range(split)]


def group_m(group_rows):
    return max(1, (group_rows or 2048) // TILE_M)


def ffma_fat(m, n, variant=-1):
    if variant >= 0:
        return bool(variant & 2)
    return cdiv(m, 128) * cdiv(n, 256) >= 96


def ffma_halves(m, n, sms, fat, variant=-1):
    on = variant < 0 or bool(variant & 1)
    bn, slots = (256, sms) if fat else (128, 2 * sms)
    rem = cdiv(m, 128) * cdiv(n, bn) % slots
    return on and rem > 0 and 2 * rem <= slots


# ==== shape generators (from the model, for a given SM count) =============================================
def width_cases(kind):
    """Forced tile width BN; M in {1, 127, 129, 3 tile rows + 5}; N at BN - 8, BN + 8, 2 BN + 8; K not a
    multiple of BK.  (m, n, k, bn)"""
    kd = KINDS[kind]
    k = 3 * kd.bk + 5 * kd.bk // 8
    return [(m, n, k, bn) for bn in kd.widths for m in (1, 127, 129, 3 * TILE_M + 5) for n in (bn - 8, bn + 8, 2 * bn + 8)]


def split_case(kind, split, sms, rounds):
    """A shape whose last round is split `split` ways into uneven parts (num_kb % split == 1), with M and N
    tails.  rounds=False: a handful of tiles, the split set by K.  rounds=True: at least two full rounds of
    tiles before the tail, the split set by the remainder of tiles over SMs.  (m, n, k, bn)"""
    kd = KINDS[kind]
    bn = kd.widths[(split - 2) % len(kd.widths)]
    num_kb = 8 * split + 1
    k = (num_kb - 1) * kd.bk + 3 * kd.bk // 8
    if not rounds:
        tm, tn = 3, 2
    else:
        def by_rem(t):
            rem = t % sms
            return rem > 0 and rem * 8 <= 1024 and min(4, sms // rem) == split
        tm, tn = min(((tm, tn) for tm in range(1, 65) for tn in range(1, 13)
                      if tm * tn // sms >= 2 and by_rem(tm * tn)), key=lambda t: (t[0] * t[1], t))
    return tm * TILE_M - 19, tn * bn - 8, k, bn


RASTER_ROWS = (128, 384, 640)      # group_m 1, 3, 5 over 8 tile rows (3 and 5 leave a ragged last group)


def raster_case(kind):
    """8 tile rows (the default 2048-row group and group_m 3 / 5 are all ragged), 3 tile columns of the widest
    tile.  int32 out: K long enough for a split tail (exact, so still bit-identical across groupings); other
    kinds: K too short for one (the split changes which tiles fold in fp32).  (m, n, k, bn)"""
    kd = KINDS[kind]
    bn = kd.widths[-1]
    num_kb = 17 if kind == "s8" else 3
    return 8 * TILE_M - 3, 2 * bn + 8, (num_kb - 1) * kd.bk + kd.bk // 2, bn


CHUNKS = (96, 100, 160)            # 3, 4 and 5 k-blocks of 32: none divides every part of a 17 / 25 k-block tile


def strict_case(sms, fat):
    """A full round of strict tiles, then a last round at most half full (issued as half tiles), M / N tails.
    (m, n, k)"""
    bn, slots = (256, sms) if fat else (128, 2 * sms)
    tm, tn = min(((tm, tn) for tm in range(2, 40) for tn in range(2, 40)
                  if tm * tn > slots and 0 < tm * tn % slots <= slots // 2), key=lambda t: (t[0] * t[1], t))
    return tm * 128 - 37, tn * bn - 12, 100


# ==== model tests (no GPU) ================================================================================
def test_schedule_model_documented_cases():
    """Facts about the schedule stated in the library's documents, on a 132-SM H100 SXM."""
    assert pick_bn(4096, 4096, 132, "bf16") == 256 and cdiv(4096, 128) * cdiv(4096, 256) % 132 == 116
    assert tc_split(4096, 4096, 4096, "bf16", 256, 132) == 1                 # 116 remainder tiles: no split
    assert pick_bn(8192, 8192, 132, "bf16") == 256 and tc_split(8192, 8192, 8192, "bf16", 256, 132) == 1   # 68
    assert tc_split(128, 128, 512, "bf16", 128, 132) == 1                   # K = 512 is 8 k-blocks: never split
    assert tc_split(128, 128, 1024, "bf16", 128, 132) == 2                  # the first K that splits
    assert tc_split(128, 128, 1 << 20, "bf16_obf16", 128, 132) == 1         # bf16 out never splits
    assert tc_split(129 * 128, 128, 1 << 20, "bf16", 128, 400) == 1         # 129 tail tiles: flag slot too small
    assert tc_split(128 * 128, 128, 1 << 20, "bf16", 128, 400) == 3
    assert ffma_fat(4096, 4096) and not ffma_fat(1024, 1024)
    assert not ffma_halves(4096, 4096, 132, True)                           # 116 remainder fat tiles: too many
    assert ffma_halves(1024, 1024, 132, False) and ffma_halves(200, 136, 132, False)


@pytest.mark.parametrize("sms", [132, 114])
def test_shape_generators_reach_every_target(sms):
    """On a 132-SM H100 SXM and a 114-SM H100 PCIe, the generated shapes reach every path the GPU tests aim at."""
    for kind in KINDS:                                   # every tile width, no split
        seen = set()
        for m, n, k, bn in width_cases(kind):
            assert pick_bn(m, n, sms, kind, force=bn) == bn and tc_split(m, n, k, kind, bn, sms) == 1
            assert k % KINDS[kind].bk and m in (1, 127, 129, 389)
            seen.add(bn)
        assert seen == set(KINDS[kind].widths)
    for kind in SPLIT_KINDS:                             # every split factor, with and without full rounds
        for split in (2, 3, 4):
            for rounds in (False, True):
                m, n, k, bn = split_case(kind, split, sms, rounds)
                tiles = cdiv(m, TILE_M) * cdiv(n, bn)
                assert tc_split(m, n, k, kind, bn, sms) == split
                assert (tiles // sms >= 2) == rounds
                assert cdiv(k, KINDS[kind].bk) % split == 1 and k % KINDS[kind].bk
                sizes = {b - a for a, b in split_parts(cdiv(k, KINDS[kind].bk), split)}
                assert len(sizes) == 2                                      # uneven parts
                assert tc_split(m, n, k, kind, bn, sms, split_tail=False) == 1
    for kind in SPLIT_KINDS:                             # every tile width of a kind meets a split
        assert {split_case(kind, s, sms, False)[3] for s in (2, 3, 4)} == set(KINDS[kind].widths)
    for kind in KINDS:                                   # ragged raster groups
        m, n, k, bn = raster_case(kind)
        tiles_m = cdiv(m, TILE_M)
        ragged = [r for r in (0,) + RASTER_ROWS if tiles_m % group_m(r)]
        assert len(ragged) >= 3
        assert tc_split(m, n, k, kind, bn, sms) == (2 if kind == "s8" else 1)
    for kind in ("bf16x3", "bf16x2", "f16x2"):           # chunks that do not divide a part
        for split in (2, 3):
            m, n, k, bn = split_case(kind, split, sms, False)
            parts = split_parts(cdiv(k, 32), split)
            for chunk in CHUNKS:
                assert any((b - a) % cdiv(chunk, 32) for a, b in parts)
    for fat in (False, True):                            # strict kernels: half tiles after a full round
        m, n, k = strict_case(sms, fat)
        bn, slots = (256, sms) if fat else (128, 2 * sms)
        assert cdiv(m, 128) * cdiv(n, bn) > slots
        for halves in (0, 1):
            v = (2 if fat else 0) | halves
            assert ffma_fat(m, n, v) == fat and ffma_halves(m, n, sms, fat, v) == bool(halves)
        assert m % 128 and n % bn and n % 4 == 0


# ==== GPU helpers ===========================================================================================
@pytest.fixture
def hooks(gemm):
    """The library's scheduling hooks, reset to their defaults after the test whatever its outcome."""
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


def mode_of(gemm, kind):
    return {"tf32": gemm.F32_TF32, "bf16x3": gemm.F32_BF16X3, "bf16x2": gemm.F32_BF16X2, "f16x2": gemm.F32_F16X2}[kind]


def pitch(cols):
    return cdiv(max(cols, 1), 16) * 16            # 16 elements: a TMA-legal pitch for every operand type


class Operands:
    """A (m x k) and B (k x n) of a kind on the device, as views of buffers with padded (TMA-legal) pitches,
    the float64 reference product, and the requant scales / bias for s8_requant."""

    def __init__(self, kind, m, n, k, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.kind, self.m, self.n, self.k = kind, m, n, k

        def make(r, c):
            if kind in ("s8", "s8_requant"):
                buf = torch.randint(-127, 128, (r, pitch(c)), device="cuda", generator=g, dtype=torch.int8)
            else:
                buf = torch.rand((r, pitch(c)), device="cuda", generator=g) * 2 - 1
                if kind in ("bf16", "bf16_obf16"):
                    buf = buf.bfloat16()
            return buf[:, :c]
        self.A, self.B = make(m, k), make(k, n)
        self.ref = self.A.double() @ self.B.double()
        self.rq = None
        if kind == "s8_requant":
            rng = np.random.default_rng(seed)
            scales = (rng.uniform(0.5, 2.0, m) * 300.0 / (127.0 ** 2 * max(k, 1) ** 0.5)).astype(np.float32)
            bias = rng.uniform(-20, 20, m).astype(np.float32)
            self.rq = (scales, bias, torch.from_numpy(scales).cuda(), torch.from_numpy(bias).cuda())

    def out(self, odd_ldc=False):
        """(buffer, m x n view): NaN / sentinel filled, optionally with an odd leading dimension."""
        dt = {"bf16_obf16": torch.bfloat16, "s8": torch.int32, "s8_requant": torch.int8}.get(self.kind, torch.float32)
        ldc = self.n + 1 + self.n % 2 if odd_ldc else self.n
        buf = torch.empty((self.m, ldc), dtype=dt, device="cuda")
        buf.fill_(float("nan") if dt.is_floating_point else 77)
        return buf, buf[:, :self.n]

    def run(self, gemm, out, accumulate=False):
        kind = self.kind
        if kind in ("bf16", "bf16_obf16"):
            gemm.gemm_bf16(self.A, self.B, out=out)
        elif kind == "s8":
            gemm.gemm_s8s32(self.A, self.B, out=out)
        elif kind == "s8_requant":
            gemm.gemm_s8s8_requant(self.A, self.B, self.rq[2], self.rq[3], out=out)
        else:
            gemm.gemm_f32(self.A, self.B, out=out, mode=mode_of(gemm, kind), accumulate=accumulate)
        return gemm.last_kernel()

    def check(self, oracle, got, c0=None, what=""):
        """got (m x n view) against the reference: int8 bit-exact, bf16 / tf32 / split modes at their tolerance."""
        kind = self.kind
        if kind == "s8":
            assert torch.equal(got.long(), self.ref.long()), what
        elif kind == "s8_requant":
            want = _libs.requant_s8(oracle, self.ref.long().int().cpu().numpy(), self.rq[0], self.rq[1])
            assert np.array_equal(got.cpu().numpy(), want), what
        elif kind == "bf16_obf16":        # one RNE rounding of the fp32 accumulator: half an ulp = 2^-9, elementwise
            t, c = self.ref, got.double()
            assert bool(((c - t).abs() <= t.abs() * 2.0 ** -8 + TOL["bf16"] * t.abs().max()).all()), what
        else:
            t = self.ref if c0 is None else self.ref + c0.double()
            err = float((got.double() - t).abs().max() / t.abs().max())
            assert err <= TOL[kind], (what, err)       # NaN (a skipped tile) fails too


def kernel_name(kind, bn):
    return f"{KINDS[kind].name}_128x{bn}"


def bits(t):
    t = t.contiguous()
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def untouched(buf, n):
    pad = buf[:, n:]
    return bool(torch.isnan(pad).all()) if pad.dtype.is_floating_point else bool((pad == 77).all())


# ==== tile widths ===========================================================================================
@gpu
@pytest.mark.parametrize("kind", ["bf16", "bf16_obf16", "tf32", "s8", "s8_requant"])
def test_tile_widths(gemm, oracle, hooks, sms, kind):
    """Each forced tile width (int8 has no 192) on M = 1 / 127 / 129 / several tile rows, N at BN - 8, BN + 8
    and 2 BN + 8, K not a multiple of BK."""
    for i, (m, n, k, bn) in enumerate(width_cases(kind)):
        assert pick_bn(m, n, sms, kind, force=bn) == bn and tc_split(m, n, k, kind, bn, sms) == 1
        hooks.b200_gemm_debug_set_bn(bn)
        op = Operands(kind, m, n, k, 100 + i)
        buf, out = op.out(odd_ldc=i % 2 == 1)
        assert op.run(gemm, out) == kernel_name(kind, bn)
        op.check(oracle, out, what=(m, n, k, bn))
        assert untouched(buf, n)


# ==== K-split tail ==========================================================================================
@gpu
@pytest.mark.parametrize("rounds", [False, True], ids=["tail_only", "after_rounds"])
@pytest.mark.parametrize("split", [2, 3, 4])
@pytest.mark.parametrize("kind", SPLIT_KINDS)
def test_split_tail(gemm, oracle, hooks, sms, kind, split, rounds):
    """The last partial round cut into `split` uneven K parts, folded into C in order.  tail_only: odd ldc (the
    scalar __ldcg fold) and, for the fp32 modes, C += A*B; after_rounds: two full rounds first.  The same call
    with whole tiles only must agree: int32 identical, fp32 within the tolerance."""
    m, n, k, bn = split_case(kind, split, sms, rounds)
    assert tc_split(m, n, k, kind, bn, sms) == split
    hooks.b200_gemm_debug_set_bn(bn)
    op = Operands(kind, m, n, k, 200 + split)
    acc = not rounds and kind in F32_KINDS
    c0 = torch.rand((m, n), device="cuda") * 2 - 1 if acc else None
    results = []
    for tail in (1, 0):
        hooks.b200_gemm_debug_set_split_tail(tail)
        buf, out = op.out(odd_ldc=not rounds)
        if acc:
            out.copy_(c0)
        assert op.run(gemm, out, accumulate=acc) == kernel_name(kind, bn)
        op.check(oracle, out, c0, what=("split_tail", tail))
        assert untouched(buf, n)
        results.append(out)
    if kind == "s8":
        assert torch.equal(results[0], results[1])
    else:
        t = op.ref if c0 is None else op.ref + c0.double()
        assert float((results[0].double() - results[1].double()).abs().max() / t.abs().max()) <= TOL[kind]


# ==== alpha / beta with a split tail ========================================================================
@gpu
@pytest.mark.parametrize("alpha,beta", [(2.5, 0.0), (-0.75, 0.5), (0.0, 2.0)])
@pytest.mark.parametrize("kind", ["tf32", "bf16x3", "f16x2"])
def test_alpha_beta_split_tail(gemm, oracle, hooks, sms, kind, alpha, beta):
    """C = alpha A*B + beta C through the fused epilogue when the tail is split: part 0 applies beta, later parts
    add alpha * partial.  beta == 0: NaN in C must not leak; alpha == 0: A and B are not read (NaN in A)."""
    m, n, k, _ = split_case(kind, 2, sms, False)
    bn = pick_bn(m, n, sms, kind)                     # the library's own choice of width
    assert tc_split(m, n, k, kind, bn, sms) == 2
    op = Operands(kind, m, n, k, 300)
    c0 = torch.rand((m, n), device="cuda") * 2 - 1
    buf, out = op.out(odd_ldc=True)
    out.copy_(c0)
    if beta == 0.0:
        out[::7, ::5] = float("nan")
    A = op.A if alpha != 0.0 else torch.full_like(op.A, float("nan"))
    gemm.gemm_f32_ex(alpha, A, op.B, beta, out, mode=mode_of(gemm, kind))
    if alpha != 0.0:
        assert gemm.last_kernel() == kernel_name(kind, bn)
    want = alpha * op.ref + beta * c0.double()
    scale = abs(alpha) * float(op.ref.abs().max()) + abs(beta) * float(c0.abs().max())
    assert bool(torch.isfinite(out).all())
    assert float((out.double() - want).abs().max()) <= TOL[kind] * scale
    assert untouched(buf, n)


# ==== raster groups =========================================================================================
@gpu
@pytest.mark.parametrize("kind", list(KINDS))
def test_raster_groups_bit_identical(gemm, oracle, hooks, sms, kind):
    """Group rows that leave a ragged last group of tile rows: the per-tile arithmetic does not depend on the
    raster order, so every grouping gives the default grouping's bits, and those match the reference."""
    m, n, k, bn = raster_case(kind)
    assert tc_split(m, n, k, kind, bn, sms) == (2 if kind == "s8" else 1)
    hooks.b200_gemm_debug_set_bn(bn)
    op = Operands(kind, m, n, k, 400)
    buf, base = op.out()
    assert op.run(gemm, base) == kernel_name(kind, bn)
    op.check(oracle, base, what="default grouping")
    for rows in RASTER_ROWS:
        hooks.b200_gemm_debug_set_group_rows(rows)
        _, out = op.out()
        assert op.run(gemm, out) == kernel_name(kind, bn)
        assert torch.equal(bits(out), bits(base)), ("group rows", rows, "group_m", group_m(rows))


# ==== chunked accumulation with a split tail =================================================================
@gpu
@pytest.mark.parametrize("split", [2, 3])
@pytest.mark.parametrize("kind", ["bf16x3", "bf16x2", "f16x2"])
def test_split_chunk_with_split_tail(gemm, oracle, hooks, sms, kind, split):
    """Two-level accumulation with chunks that do not divide a split part's K."""
    m, n, k, bn = split_case(kind, split, sms, False)
    assert tc_split(m, n, k, kind, bn, sms) == split
    op = Operands(kind, m, n, k, 500 + split)
    for chunk in CHUNKS:
        hooks.b200_gemm_debug_set_split_chunk(chunk, chunk)
        buf, out = op.out(odd_ldc=True)
        assert op.run(gemm, out) == kernel_name(kind, bn)
        op.check(oracle, out, what=("chunk", chunk))


@gpu
def test_split_chunk_negative_restores_defaults(gemm, hooks):
    """b200_gemm_debug_set_split_chunk(-1, -1) brings back the built-in chunks of all three split modes."""
    g = torch.Generator(device="cuda").manual_seed(9)
    A = torch.rand((256, 4096), device="cuda", generator=g) * 2 - 1
    B = torch.rand((4096, 384), device="cuda", generator=g) * 2 - 1
    modes = (gemm.F32_BF16X3, gemm.F32_BF16X2, gemm.F32_F16X2)
    before = [gemm.gemm_f32(A, B, mode=md) for md in modes]
    hooks.b200_gemm_debug_set_split_chunk(64, 64)
    changed = [gemm.gemm_f32(A, B, mode=md) for md in modes]
    assert not all(torch.equal(x, y) for x, y in zip(before, changed))
    hooks.b200_gemm_debug_set_split_chunk(-1, -1)
    for md, ref in zip(modes, before):
        assert torch.equal(gemm.gemm_f32(A, B, mode=md), ref), md


# ==== strict FFMA kernels ===================================================================================
@gpu
@pytest.mark.parametrize("halves", [1, 0], ids=["halves", "whole"])
@pytest.mark.parametrize("fat", [False, True], ids=["128x128", "fat_128x256"])
def test_strict_ffma_schedules_bit_exact(gemm, oracle, hooks, sms, fat, halves):
    """Both strict kernels with the last round as half tiles or as whole tiles, M / N tails, odd ldc, C = A*B and
    C += A*B: one sequential FMA chain per element, bit-exact against the oracle."""
    m, n, k = strict_case(sms, fat)
    variant = (2 if fat else 0) | halves
    assert ffma_fat(m, n, variant) == fat and ffma_halves(m, n, sms, fat, variant) == bool(halves)
    hooks.b200_gemm_debug_set_ffma_variant(variant)
    a, b, c0 = _libs.gen_f32(oracle, m, k, 601), _libs.gen_f32(oracle, k, n, 602), _libs.gen_f32(oracle, m, n, 603)
    A, B = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    name = "ffma_fat_128x256x32_tma" if fat else "ffma_128x128x32_tma"
    ldc = n + 1 + n % 2
    buf = torch.full((m, ldc), float("nan"), device="cuda")
    gemm.gemm_f32(A, B, out=buf[:, :n], mode=gemm.F32_STRICT)
    assert gemm.last_kernel() == name
    assert np.array_equal(buf[:, :n].cpu().numpy(), _libs.ref_f32_fma(oracle, a, b))
    buf[:, :n] = torch.from_numpy(c0).cuda()
    gemm.gemm_f32(A, B, out=buf[:, :n], mode=gemm.F32_STRICT, accumulate=True)
    assert gemm.last_kernel() == name
    assert np.array_equal(buf[:, :n].cpu().numpy(), _libs.ref_f32_fma(oracle, a, b, c0))
    assert untouched(buf, n)


# ==== two streams ===========================================================================================
@gpu
def test_two_streams_bit_identical(gemm, hooks, sms):
    """TF32 and F16X2 GEMMs with different operands interleaved on two streams without host synchronisation
    (shared workspace, double-buffered column maxima, rotating flag slots, split tails) give the bits of the
    same calls on one stream."""
    hooks.b200_gemm_debug_set_bn(128)
    calls = []
    for i, (kind, split) in enumerate([("tf32", 2), ("f16x2", 3)] * 3):
        m, n, k, _ = split_case(kind, split, sms, i >= 2)
        assert tc_split(m, n, k, kind, 128, sms) == split
        calls.append(Operands(kind, m, n, k, 700 + i))
    one = []
    for op in calls:
        _, out = op.out()
        op.run(gemm, out)
        one.append(out)
    torch.cuda.synchronize()
    cur = torch.cuda.current_stream()
    streams = (torch.cuda.Stream(), torch.cuda.Stream())
    two = [op.out()[1] for op in calls]
    for s in streams:
        s.wait_stream(cur)
    for i, (op, out) in enumerate(zip(calls, two)):
        with torch.cuda.stream(streams[i % 2]):
            op.run(gemm, out)
    for s in streams:
        cur.wait_stream(s)
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(one, two)):
        assert torch.equal(x, y), (i, calls[i].kind)


# ==== alpha / beta extremes ===================================================================================
EXTREMES = [(1e-20, 1e20), (1e20, 1e-20), (2.0 ** -70, 2.0 ** 70)]


@gpu
@pytest.mark.parametrize("alpha,beta", EXTREMES, ids=["tiny_alpha", "tiny_beta", "pow2"])
@pytest.mark.parametrize("route", ["strict", "auto_small", "unaligned_strict", "unaligned_tf32",
                                   "tf32", "bf16x3", "bf16x2", "f16x2"])
def test_alpha_beta_extremes(gemm, oracle, route, alpha, beta):
    """beta / alpha far outside the fp32 range: the answer alpha A*B + beta C is finite and every route returns
    it within its tolerance (cuBLAS's contract; pre-scaling C by beta / alpha overflows)."""
    m, n, k = 200, 136, 264
    a, b, c0 = _libs.gen_f32(oracle, m, k + 1, 61), _libs.gen_f32(oracle, k + 1, n + 1, 62), _libs.gen_f32(oracle, m, n, 63)
    Ad, Bd = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    if route.startswith("unaligned"):
        A, B = Ad[:, 1:], Bd[1:, 1:]                   # misaligned bases: no TMA
        a_use, b_use = a[:, 1:], b[1:, 1:]
    else:
        A, B = Ad[:, :k].contiguous(), Bd[:k, :n].contiguous()
        a_use, b_use = a[:, :k], b[:k, :n]
    mode, name, tol = {
        "strict": (gemm.F32_STRICT, "ffma_128x128x32_tma", TOL_STRICT),
        "auto_small": (gemm.F32_AUTO, "ffma_128x128x32_tma", TOL_STRICT),
        "unaligned_strict": (gemm.F32_STRICT, "generic_f32_64x64", TOL_STRICT),
        "unaligned_tf32": (gemm.F32_TF32, "generic_f32_64x64", TOL_STRICT),
        "tf32": (gemm.F32_TF32, "tc_tf32_128x128", TOL["tf32"]),
        "bf16x3": (gemm.F32_BF16X3, "tc_bf16x3_128x128", TOL["bf16x3"]),
        "bf16x2": (gemm.F32_BF16X2, "tc_bf16x2_128x128", TOL["bf16x2"]),
        "f16x2": (gemm.F32_F16X2, "tc_f16x2_128x128", TOL["f16x2"]),
    }[route]
    ldc = n + 1
    buf = torch.full((m, ldc), float("nan"), device="cuda")
    buf[:, :n] = torch.from_numpy(c0).cuda()
    gemm.gemm_f32_ex(alpha, A, B, beta, buf[:, :n], mode=mode)
    assert gemm.last_kernel() == name
    got = buf[:, :n].cpu().numpy().astype(np.float64)
    al, be = float(np.float32(alpha)), float(np.float32(beta))
    ab = _libs.ref_f64(oracle, np.ascontiguousarray(a_use), np.ascontiguousarray(b_use))
    want = al * ab + be * c0.astype(np.float64)
    assert np.isfinite(got).all(), "alpha/beta overflowed"
    scale = abs(al) * np.abs(ab).max() + abs(be) * np.abs(c0).max()
    assert np.abs(got - want).max() <= tol * scale, np.abs(got - want).max() / scale
    assert bool(torch.isnan(buf[:, n:]).all())
