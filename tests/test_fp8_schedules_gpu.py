"""Every FP8 kernel's persistent schedule against exact references: several tiles per CTA, K through the stage ring,
ragged raster groups, every tile width and every stacking.

gemm_tc_fp8_kernel is persistent: CTA b takes work tiles b, b + grid, b + 2 grid, ..., each tile's (mb, nb) from
tile_coords and its raster groups.  The TMA thread, the blockwise scale loaders and both consumer warpgroups each carry
their own copy of the ring's stage index and phase bit from one tile to the next, and the blockwise loaders recompute
the tile order on their own.  If one of them gets out of step the kernel reads the wrong stage or the wrong scales, and
its output is slightly wrong or comes from a neighbouring tile.  So every case here has at least two full rounds of tiles
plus a partial one, more k-blocks than stages (a CTA starts a later tile in the middle of the ring with the phase bit
flipped), and at least 17 tile rows in one matrix or group (the default 2048-row raster group is ragged, as are the
forced group rows 384 and 640).  The shapes come from a Python restatement of the host's choices (the schedule model
below), read with the device's SM count; every GPU case asserts that the model says it reaches its targets, and that
the schedule the library reports is the model's.

The results are exact, so every case is compared bit for bit:
- integer operands in [-2, 2] decode to the same values in e4m3 and e5m2, and every partial sum is an integer below 2^13
  (K <= 2047), which the tensor core's >= 14 retained bits (test_fp8_gpu.RETAINED_BITS) keep exactly in fast mode;
  promoted and blockwise chunks are exact and their fp32 running sums are integers below 2^24.  One float64 product on
  the device therefore serves all three operand pairs;
- the float32 contract on that product is test_fp8_gpu.oracle (rowwise: (acc * sa) * sb + bias, one rounding each),
  test_fp8_blockwise_gpu's FMA-chain oracle (blockwise, random fp32 scales), and test_fp8_out_gpu's quantisers (FP8 C).
Outputs start as NaN (16/32-bit C) or a sentinel byte (FP8 C, scale_c), the operands' padding holds FP8 NaN bytes, and
the whole buffer is compared, fences included.

The CPU tests show that the data discriminates: no two output tiles of a case are equal, a blockwise tile computed with
a neighbouring k-block's, row block's or column block's scales changes, and neighbouring dynamic scale blocks differ.
So a tile stored at the wrong place, a scale loader one step out, or a scale stored in the wrong slot cannot pass.  A
case-table test checks that the GPU cases reach all 159 FP8 kernels."""
import functools

import numpy as np
import pytest

import test_batched_gpu as bt
import test_fp8_blockwise_gpu as bw
import test_fp8_blockwise_grouped_gpu as bfg
import test_fp8_gpu as f8
import test_fp8_grouped_gpu as fg
import test_fp8_out_gpu as fo
import test_grouped_gpu as gg
import test_tile_schedules_gpu as ts
import test_transposed_ops_gpu as tr
from test_transposed_ops_gpu import hooks, sms  # noqa: F401  (fixtures: scheduling hooks reset, SM count)

try:
    import torch
except ImportError:          # the model and discrimination tests need no torch
    torch = None

gpu = pytest.mark.gpu
E4M3, E5M2 = f8.E4M3, f8.E5M2
OUT_F32, OUT_BF16, OUT_F16 = f8.OUT_F32, f8.OUT_BF16, f8.OUT_F16
OUTS = (OUT_F32, OUT_BF16, OUT_F16)
PAIRS, PAIR_NAME, OUT_NAME = f8.PAIRS, f8.PAIR_NAME, f8.OUT_NAME
CTS = (E4M3, E5M2)
RECIPES = bw.RECIPES
cdiv = ts.cdiv


# ==== schedule model ====================================================================================================
# A restatement of the FP8 host choices of csrc/capi.cu:
#   tc_fp8                   -> fp8_width()   fast: pick_bn over {256, 192, 128} (FP8 C: {256, 128}; a forced 192 falls
#                                             back to the heuristic); promoted and blockwise: always 128
#   Width<BN>                -> STAGES         4, 5 and 6 stages at BN = 256, 192 and 128
#   launch_tc                -> schedule()     one CTA per SM, grid = min(tiles, SMs); FP8 never splits K; a grouped
#                                             call launches for its tile bound (test_grouped_gpu.tile_bound)
#                               group_m        rows per raster group / 128, 2048 rows by default (ts.group_m)
# and of gemm_tc_fp8_kernel: CTA b walks work tiles b, b + grid, ...; the i-th of them starts at ring stage
# (i * num_kb) mod STAGES with phase bit floor(i * num_kb / STAGES) mod 2 (ring_start).  If a heuristic there changes,
# update it here: the generators then still aim at every target, and the model assertions of each GPU case fail instead
# of quietly losing coverage.
BK = 128                                  # K elements per stage: one 128-byte swizzled row of FP8
STAGES = {256: 4, 192: 5, 128: 6}
WIDTHS = (256, 192, 128)
RASTER_ROWS = ts.RASTER_ROWS              # forced group rows 128, 384, 640: group_m 1, 3, 5
RAGGED_ROWS = (0, 384, 640)               # the default and the forced rows that leave a ragged last group
EXACT_FAST_K = (2 ** 13 - 1) // 4         # 2047: |partial sums| <= 4 K stay below 2^13 with operands in [-2, 2]


def fp8_width(stack, sizes, n, sms, accum, force=0, fp8_out=False):
    """The tile width of an FP8 call: stack "none" (one matrix of sizes[0] rows), "bat" (len(sizes) entries of
    sizes[0] rows) or "grp" (groups of sizes rows); accum "fast", "promoted" or "blk"; force: the set_bn hook."""
    if accum != "fast":
        return 128
    if stack == "none":                   # ts's int8 kind has exactly the widths {256, 128} of an FP8 C
        return ts.pick_bn(sizes[0], n, sms, "s8" if fp8_out else "bf16", force)
    if stack == "bat":
        return bt.bat_pick_bn(sizes[0], n, len(sizes), sms, force)
    return gg.grp_pick_bn(sum(sizes), n, len(sizes), sms, force)


def launched_tiles(stack, sizes, n, bn):
    """The tiles the host sizes the grid for: every entry's, or a grouped call's bound."""
    rows = gg.tile_bound(sum(sizes), len(sizes)) if stack == "grp" else sum(cdiv(s, 128) for s in sizes)
    return rows * cdiv(n, bn)


def walked_tiles(sizes, n, bn):
    """The tiles the CTAs walk: each entry's or group's own tile rows."""
    return sum(cdiv(s, 128) for s in sizes) * cdiv(n, bn)


def schedule(stack, sizes, n, bn, sms):
    """(tiles, split, full_tiles, ctas) that b200_gemm_debug_last_schedule reports: whole tiles, no K split."""
    tiles = launched_tiles(stack, sizes, n, bn)
    return tiles, 1, tiles, min(tiles, sms)


def ring_start(i, num_kb, stages):
    """(stage, phase) at which a CTA's i-th tile starts in the ring of `stages` stages."""
    return i * num_kb % stages, i * num_kb // stages % 2


def reach(stack, sizes, n, k, bn, sms):
    """The targets a case reaches: rounds (two full rounds of tiles and a partial one), mid_ring (a later tile of a CTA
    starts at a non-zero stage with the phase bit flipped), ragged (group rows whose last raster group of the largest
    matrix / group is ragged)."""
    tiles = walked_tiles(sizes, n, bn)
    grid = min(launched_tiles(stack, sizes, n, bn), sms)
    num_kb, st = cdiv(k, BK), STAGES[bn]
    starts = [ring_start(i, num_kb, st) for i in range(1, cdiv(tiles, grid))]
    tm = max(cdiv(s, 128) for s in sizes)
    return {"rounds": tiles // grid >= 2 and tiles % grid != 0,
            "mid_ring": num_kb > st and num_kb % st != 0 and any(s != 0 and ph == 1 for s, ph in starts),
            "ragged": {r for r in (0,) + RASTER_ROWS if tm >= 17 and tm % ts.group_m(r)}}


def reaches_all(stack, sizes, n, k, bn, sms):
    t = reach(stack, sizes, n, k, bn, sms)
    return t["rounds"] and t["mid_ring"] and t["ragged"] >= set(RAGGED_ROWS)


# ==== shape generators (from the model, for a given SM count) ============================================================
TM = 17                                   # tile rows of the largest matrix / group: 17 % 16, % 3 and % 5 are all non-zero
M_BIG = TM * 128 - 19                     # 2157 rows: an M tail
K = 7 * BK - 48                           # 848: 7 k-blocks (more than 4, 5 and 6 stages, a multiple of none), a K tail
GROUPS = [300, 0, 1, M_BIG, 0, 517, 129]  # empty groups, a 1-row group, a group of more than 2048 rows
BATCH = 2
# family: (stack, rows per entry, tile widths its kernels use)
FAMILIES = {
    "single": ("none", [M_BIG], WIDTHS),              # b200_gemm_fp8 (fast and promoted), _q8 fast and promoted
    "single_blk": ("none", [M_BIG], (128,)),          # b200_gemm_fp8_blockwise, _blockwise_q8
    "grp": ("grp", GROUPS, WIDTHS),
    "grp_blk": ("grp", GROUPS, (128,)),
    "bat": ("bat", [M_BIG] * BATCH, WIDTHS),
    "bat_blk": ("bat", [M_BIG] * BATCH, (128,)),
}


@functools.lru_cache(maxsize=None)
def family_shape(family, sms):
    """(stack, sizes, n, k): the narrowest N (a tail at every width) at which every width of the family reaches every
    target on `sms` SMs."""
    stack, sizes, widths = FAMILIES[family]
    for tn in range(1, 200):
        n = tn * max(widths) - 8
        if all(n % bn and reaches_all(stack, sizes, n, K, bn, sms) for bn in widths):
            return stack, tuple(sizes), n, K
    raise AssertionError(f"no shape reaches every target for {family} on {sms} SMs")


# ==== model tests (no GPU) ================================================================================================
def test_schedule_model_documented_facts():
    """Facts about the FP8 schedule stated in csrc/capi.cu and DESIGN §4.7, on a 132-SM H100 SXM."""
    # fp32 C, a partial last round and a long K: the FP8 kernels never split K; the 16-bit model would split 4 ways
    assert schedule("none", [384], 256, 128, 132) == (6, 1, 6, 6)
    assert ts.tc_split(384, 256, 8192, "bf16", 128, 132) == 4
    # promoted and blockwise are 128 wide whatever the hook says; FP8 C has no 192-wide tile
    for accum in ("promoted", "blk"):
        assert fp8_width("none", [4096], 4096, 132, accum, force=256) == 128
    assert fp8_width("none", [4096], 4096, 132, "fast", force=192) == 192
    assert fp8_width("none", [4096], 4096, 132, "fast", force=192, fp8_out=True) == \
        fp8_width("none", [4096], 4096, 132, "fast", fp8_out=True) == 256
    assert fp8_width("none", [256], 1024, 132, "fast", force=192, fp8_out=True) == 128   # 8 tiles: narrow wins
    # stacked widths and schedules: over the whole batch, or over a grouped call's tile bound
    assert fp8_width("bat", [512] * 128, 512, 132, "fast") == 256 and fp8_width("bat", [512], 512, 132, "fast") == 128
    assert schedule("grp", [300, 0, 1], 200, 128, 132) == gg.grp_schedule(301, 200, 3, 128, 132) == (12, 1, 12, 12)
    assert schedule("bat", [300] * 4, 200, 192, 132) == (24, 1, 24, 24)
    # the ring: 7 k-blocks put a CTA's second tile mid-ring with the phase flipped at every width
    assert [ring_start(1, 7, STAGES[bn]) for bn in WIDTHS] == [(3, 1), (2, 1), (1, 1)]
    assert ring_start(0, 7, 6) == (0, 0) and ring_start(2, 7, 5) == (4, 0) and ring_start(6, 4, 6) == (0, 0)
    # 3 k-blocks (test_many_groups) or 9 (test_grouped_k_tails, one round) never start a later tile mid-ring flipped
    assert not reach("grp", [128] * 200, 136, 3 * 128, 128, 132)["mid_ring"]
    assert not reach("grp", [300] * 4, 200, 1040, 128, 132)["rounds"]
    # the raster groups: 2048 rows by default; 17 tile rows leave a ragged last group there and at 384 / 640 rows
    assert ts.group_m(0) == 16 and reach("none", [M_BIG], 256, K, 128, 132)["ragged"] == set(RAGGED_ROWS)
    assert reach("none", [2048], 256, K, 128, 132)["ragged"] == set()


@pytest.mark.parametrize("sms", [132, 114])
def test_shape_generators_reach_every_target(sms):
    """On a 132-SM H100 SXM and a 114-SM H100 PCIe, every family's shape reaches every target at every width it uses,
    with M, N and K tails, and inside the exactness bound of its operands."""
    for family, (stack, _, widths) in FAMILIES.items():
        _, sizes, n, k = family_shape(family, sms)
        for bn in widths:
            t = reach(stack, sizes, n, k, bn, sms)
            assert t["rounds"] and t["mid_ring"] and t["ragged"] == set(RAGGED_ROWS), (family, bn, t)
            assert launched_tiles(stack, sizes, n, bn) // sms >= 2 and n % bn, (family, bn)
        assert max(sizes) % 128 and k % BK and cdiv(k, BK) > max(STAGES.values())
        assert k <= EXACT_FAST_K                          # fast accumulation: every partial sum below 2^13
        assert 4 * k < 2 ** 24                            # promoted / blockwise: exact fp32 running sums
        if stack == "grp":
            assert 0 in sizes and 1 in sizes and max(sizes) > 2048
    assert EXACT_FAST_K == 2047 and 4 * EXACT_FAST_K < 2 ** 13 <= 4 * (EXACT_FAST_K + 1)


# ==== case tables: what the GPU tests run =================================================================================
MODES = ("fast256", "fast192", "fast128", "promoted")
Q8_ACCUMS = ("fast256", "fast128", "promoted", "blk")


def accum_of(mode):
    return ("fast", int(mode[4:])) if mode.startswith("fast") else (mode, 0)


def rowwise_scaling(pair, o, mode):
    """Half the single-matrix cases take rowwise power-of-two scales and a bias, the others tensorwise scales."""
    return "row" if (PAIRS.index(pair) + OUTS.index(o) + MODES.index(mode)) % 2 == 0 else "tensor"


SINGLE_CASES = [(pair, o, mode) for o in OUTS for mode in MODES for pair in PAIRS]
BLK_CASES = [(pair, o, RECIPES[i]) for i, o in enumerate(OUTS) for pair in PAIRS]
Q8_CASES = [(pair, ct, accum) for ct in CTS for accum in Q8_ACCUMS for pair in PAIRS]
STACK_CASES = [(stack, pair, o, mode) for stack in ("grp", "bat") for o in OUTS for mode in MODES for pair in PAIRS]
# a grouped A is always 1 x 128: the grouped entry point takes two recipes, the batched one three
STACK_BLK_RECIPES = {"grp": [(1, 128), (1, 1), (1, 128)], "bat": RECIPES}
STACK_BLK_CASES = [(stack, pair, o, STACK_BLK_RECIPES[stack][i]) for stack in ("grp", "bat") for i, o in enumerate(OUTS)
                   for pair in PAIRS]


def suffix(accum, bn):
    return {"promoted": "_acc_128x128", "blk": "_blk_128x128"}.get(accum, f"_128x{bn}")


def kernel_name(pair, out, accum, bn, stack="none"):
    """out: an OUT_* type, or "oe4m3" / "oe5m2" for an FP8 C."""
    o = out if isinstance(out, str) else OUT_NAME[out]
    return f"tc_{PAIR_NAME[pair]}_{o}" + ("" if stack == "none" else "_" + stack) + suffix(accum, bn)


def case_kernels():
    """The kernel names the case tables reach, by family."""
    def name(pair, out, mode, stack="none"):
        accum, bn = accum_of(mode)
        return kernel_name(pair, out, accum, bn or 128, stack)
    return {
        "single": {name(p, o, md) for p, o, md in SINGLE_CASES},
        "blockwise": {name(p, o, "blk") for p, o, _ in BLK_CASES},
        "q8": {name(p, fo.CT_NAME[ct], acc) for p, ct, acc in Q8_CASES},
        "stacked": {name(p, o, md, st) for st, p, o, md in STACK_CASES},
        "stacked_blk": {name(p, o, "blk", st) for st, p, o, _ in STACK_BLK_CASES},
    }


def test_cases_cover_every_fp8_kernel():
    """The GPU cases below (each asserts last_kernel() against these names) reach every FP8 kernel: 36 b200_gemm_fp8, 9
    blockwise, 24 FP8-output, 72 stacked rowwise and 18 stacked blockwise, every recipe of each entry point."""
    pn = [PAIR_NAME[p] for p in PAIRS]
    on = [OUT_NAME[o] for o in OUTS]
    widths = ["_128x256", "_128x192", "_128x128", "_acc_128x128"]
    want = {
        "single": {f"tc_{p}_{o}{w}" for p in pn for o in on for w in widths},
        "blockwise": {f"tc_{p}_{o}_blk_128x128" for p in pn for o in on},
        "q8": {f"tc_{p}_{c}{w}" for p in pn for c in ("oe4m3", "oe5m2")
               for w in ("_128x256", "_128x128", "_acc_128x128", "_blk_128x128")},
        "stacked": {f"tc_{p}_{o}_{s}{w}" for p in pn for o in on for s in ("grp", "bat") for w in widths},
        "stacked_blk": {f"tc_{p}_{o}_{s}_blk_128x128" for p in pn for o in on for s in ("grp", "bat")},
    }
    got = case_kernels()
    assert got == want
    assert [len(v) for v in got.values()] == [36, 9, 24, 72, 18] and len(set().union(*got.values())) == 159
    assert {fg.kernel_name(*p, o, s, m if m == "acc" else m) for s in ("grp", "bat") for p in PAIRS for o in OUTS
            for m in ("acc", 256, 192, 128)} == got["stacked"]
    assert {bfg.kernel_name(*p, o, s) for s in ("grp", "bat") for p in PAIRS for o in OUTS} == got["stacked_blk"]
    assert {r for _, _, r in BLK_CASES} == set(RECIPES) == set(STACK_BLK_RECIPES["bat"])
    assert set(STACK_BLK_RECIPES["grp"]) == {(1, b) for b in bfg.B_BLOCKS}


# ==== problems: integer operands, scales, exact products ==================================================================
class Problem:
    """One family's operands on the host: A (the entries' rows stacked, rows x k) and each entry's B^T (E x n x k), integer
    values in [-2, 2] as float32; rowwise power-of-two scales (exact), rowwise random-significand scales (FP8 C), a bias
    of bf16 (and fp16) values, blockwise random fp32 scales per recipe.  All drawn from the seed."""

    def __init__(self, family, sms, seed):
        self.stack, self.sizes, self.n, self.k = family_shape(family, sms)
        self.family, self.seed = family, seed
        self.E = len(self.sizes)
        self.rows = sum(self.sizes)
        self.starts = [0] + list(np.cumsum(self.sizes))
        rng = np.random.default_rng(seed)
        n, k = self.n, self.k
        self.a = rng.integers(-2, 3, (self.rows, k)).astype(np.float32)
        self.bt = rng.integers(-2, 3, (self.E, n, k)).astype(np.float32)
        self.sa_pow2 = f8.pow2_scales(rng, self.rows)
        self.sb_pow2 = f8.pow2_scales(rng, self.E * n).reshape(self.E, n)
        self.s_tensor = f8.pow2_scales(rng, 2)
        self.sa_rand = bw.random_scales(rng, (self.rows,))
        self.sb_rand = bw.random_scales(rng, (self.E, n))
        self.bias = f8.round_out(rng.integers(-64, 65, n).astype(np.float32) / 8, OUT_BF16)   # exact in fp16 too
        self.s_r = float(bw.random_scales(rng, (1,))[0])
        # C: entry e's rows start at c_row0[e]; one NaN row after each batch entry / after the last group, 8 columns
        self.ldc = n + 8
        if self.stack == "bat":
            m = self.sizes[0]
            self.c_row0 = [e * (m + 1) for e in range(self.E)]
            self.c_rows, self.stride_c = self.E * (m + 1), (m + 1) * self.ldc
        else:
            self.c_row0, self.c_rows = self.starts[:-1], self.rows + 1

    def entries(self):
        """(e, lo, hi): each non-empty entry's rows of the stacked A."""
        return [(e, lo, hi) for e, (lo, hi) in enumerate(zip(self.starts[:-1], self.starts[1:])) if hi > lo]

    @functools.lru_cache(maxsize=None)
    def blk_scales(self, recipe):
        """Random fp32 block scales in the call's layout: one matrix (R, q) and (q, C); grouped (total_m, q) and
        (G, q, C); batched (E, R, q) and (E, q, C)."""
        a_blk, b_blk = recipe
        rng = np.random.default_rng([self.seed, a_blk, b_blk])
        q, m = cdiv(self.k, 128), self.sizes[0]
        cols = cdiv(self.n, 128) if b_blk == 128 else self.n
        rows = m if a_blk == 1 else cdiv(m, 128)
        if self.stack == "none":
            return bw.random_scales(rng, (rows, q)), bw.random_scales(rng, (q, cols))
        if self.stack == "grp":
            assert a_blk == 1
            return bw.random_scales(rng, (self.rows, q)), bw.random_scales(rng, (self.E, q, cols))
        return bw.random_scales(rng, (self.E, rows, q)), bw.random_scales(rng, (self.E, q, cols))

    def entry_blk_scales(self, recipe, e, lo, hi):
        sa, sb = self.blk_scales(recipe)
        if self.stack == "none":
            return sa, sb
        if self.stack == "grp":
            return sa[lo:hi], sb[e]
        return sa[e], sb[e]

    def sampled_rows(self):
        """The first row of every tile row of every entry (rows of the stacked A), and their entries."""
        return [(e, lo + 128 * mb) for e, lo, hi in self.entries() for mb in range(cdiv(hi - lo, 128))]

    def place(self, want):
        """want (rows x n, float32) at its place in a NaN-filled C buffer (c_rows x ldc)."""
        buf = np.full((self.c_rows, self.ldc), np.nan, np.float32)
        for e, lo, hi in self.entries():
            r0 = self.c_row0[e]
            buf[r0:r0 + hi - lo, :self.n] = want[lo:hi]
        return buf


@functools.lru_cache(maxsize=None)
def problem(family, sms):
    return Problem(family, sms, seed=sorted(FAMILIES).index(family) + 10)


# ---- the float32 contract on the exact products (the existing oracles) --------------------------------------------------
def rowwise_want(P, acc, sa, sb, bias, o, rows=None):
    """test_fp8_gpu.oracle per entry: acc (rows x n, float64, exact), sa per row of A, sb (E x n).  rows: a subset of A's
    rows (sampled_rows), acc holding just those."""
    if rows is None:
        return np.concatenate([f8.oracle(None, None, sa[lo:hi], sb[e], bias, o, acc=acc[lo:hi])
                               for e, lo, hi in P.entries()])
    return np.stack([f8.oracle(None, None, sa[r:r + 1], sb[e], bias, o, acc=acc[i:i + 1])[0]
                     for i, (e, r) in enumerate(rows)])


def blk_want(P, recipe, o, bias=None, rows=None, tweak=None):
    """test_fp8_blockwise_gpu's FMA-chain oracle per entry.  rows: a subset of A's rows (sampled_rows).  tweak(e, lo, hi,
    sa_full, sb_full) -> (sa_full, sb_full): the scales a kernel out of step would use."""
    out = []
    for e, lo, hi in P.entries():
        sa_e, sb_e = P.entry_blk_scales(recipe, e, lo, hi)
        sa_full, sb_full = bw.expand_scales(sa_e, sb_e, recipe, hi - lo, P.n)
        if tweak is not None:
            sa_full, sb_full = tweak(e, lo, hi, sa_full, sb_full)
        sel = np.arange(hi - lo) if rows is None else np.array([r - lo for ee, r in rows if ee == e], int)
        out.append(bw.oracle_blockwise(P.a[lo + sel], P.bt[e].T, sa_full[sel], sb_full, bias, o))
    return np.concatenate(out)


def host_product(P, rows=None):
    """The exact products on the host, as float64: a float32 matmul is exact, every partial sum being an integer below
    2^13.  rows: a subset of A's rows (sampled_rows), else every entry's rows."""
    if rows is None:
        return np.concatenate([P.a[lo:hi] @ P.bt[e].T for e, lo, hi in P.entries()]).astype(np.float64)
    return np.stack([P.a[r] @ P.bt[e].T for e, r in rows]).astype(np.float64)


def q8_v(P, acc=None, rows=None):
    """v of the FP8-output cases, before the activation: rowwise random-significand scales (one matrix, acc its exact
    product) or the (1 x 128, 128 x 128) blockwise recipe, then the bias."""
    if P.family == "single_blk":
        return blk_want(P, (1, 128), OUT_F32, P.bias, rows=rows)
    acc = host_product(P, rows) if acc is None else acc
    return rowwise_want(P, acc, P.sa_rand, P.sb_rand, P.bias, OUT_F32, rows=rows)


# ==== discrimination (no GPU) =============================================================================================
def tile_segments(P, vals, rows, bn):
    """{(entry, row, nb): bytes of the tile's first row} from vals (one row per sampled row), NaN-padded to bn columns."""
    pad = np.full((len(rows), cdiv(P.n, bn) * bn), np.nan, np.float32)
    pad[:, :P.n] = vals
    return {(e, r, nb): pad[i, nb * bn:(nb + 1) * bn].tobytes() for i, (e, r) in enumerate(rows)
            for nb in range(cdiv(P.n, bn))}


def expected_first_rows(P, rows):
    """The fp32-C values of every family's exact cases at the sampled rows."""
    if P.family.endswith("_blk"):
        return blk_want(P, (1, 128), OUT_F32, P.bias if P.stack == "none" else None, rows=rows)
    acc = host_product(P, rows)
    bias = P.bias if P.stack == "none" else None
    return rowwise_want(P, acc, P.sa_pow2, P.sb_pow2, bias, OUT_F32, rows=rows)


@pytest.mark.parametrize("sms", [132, 114])
def test_no_two_tiles_are_equal(sms):
    """In every family's data, at every width it uses, the first rows of any two output tiles differ (so the tiles do):
    a tile stored at the wrong (mb, nb), or into the wrong entry, cannot match."""
    for family, (_, _, widths) in FAMILIES.items():
        P = problem(family, sms)
        rows = P.sampled_rows()
        vals = [expected_first_rows(P, rows)]
        if family in ("single", "single_blk"):
            vals.append(fo.relu_np(q8_v(P, rows=rows)))
        for v in vals:
            for bn in widths:
                seg = tile_segments(P, v, rows, bn)
                assert len(set(seg.values())) == len(seg), (family, bn)


def neighbour(idx, lo, hi):
    """idx + 128 (the next tile's row / column), or idx - 128 where that is past the end."""
    return np.where(idx + 128 < hi, idx + 128, idx - 128)


def scale_tweaks(P, recipe):
    """What a blockwise scale loader out of step would use instead of the right scales: the k-block before or after
    (A's or B's), or the neighbouring tile's row scales (rows of the stacked A for a grouped call, of the entry
    otherwise) or column scales."""
    def kb(which, shift):
        def f(e, lo, hi, sa, sb):
            return (np.roll(sa, shift, axis=1), sb) if which == "a" else (sa, np.roll(sb, shift, axis=0))
        return f

    def row(e, lo, hi, sa, sb):
        if P.stack == "grp":                         # a grouped A is 1 x 128: its scales are one row per stacked row
            return P.blk_scales(recipe)[0][neighbour(np.arange(lo, hi), 0, P.rows)], sb
        return sa[neighbour(np.arange(hi - lo), 0, hi - lo)], sb

    def col(e, lo, hi, sa, sb):
        return sa, sb[:, neighbour(np.arange(P.n), 0, P.n)]
    return {"a kb-1": kb("a", 1), "a kb+1": kb("a", -1), "b kb-1": kb("b", 1), "b kb+1": kb("b", -1),
            "row tile": row, "column tile": col}


BLK_FAMILY_RECIPES = {"single_blk": RECIPES, "grp_blk": STACK_BLK_RECIPES["grp"][:2], "bat_blk": RECIPES}


@pytest.mark.parametrize("sms", [132, 114])
def test_blockwise_scales_out_of_step_change_every_tile(sms):
    """For every blockwise family and recipe the GPU tests use: the oracle with any one of the scale mix-ups of
    scale_tweaks differs from the right one in every output tile (in the tile's first row), so a scale loader or a
    consumer one k-block or one tile out of step cannot pass.  As test_fp8_blockwise_gpu's exact test shows for two
    roundings."""
    for family, recipes in BLK_FAMILY_RECIPES.items():
        P = problem(family, sms)
        rows = P.sampled_rows()
        for recipe in recipes:
            base = tile_segments(P, blk_want(P, recipe, OUT_F32, rows=rows), rows, 128)
            for what, tweak in scale_tweaks(P, recipe).items():
                seg = tile_segments(P, blk_want(P, recipe, OUT_F32, rows=rows, tweak=tweak), rows, 128)
                same = [t for t in base if seg[t] == base[t]]
                assert not same, (family, recipe, what, same[:4])


@pytest.mark.parametrize("sms", [132, 114])
def test_neighbouring_dynamic_scales_differ(sms):
    """The FP8-output cases' dynamic mode: every (row, 128-column) block's scale d differs from its neighbours' in the
    row and in the column, for both C types, so a scale stored in a neighbouring slot cannot pass."""
    for family in ("single", "single_blk"):
        v = fo.relu_np(q8_v(problem(family, sms)))
        for ct in CTS:
            d = fo.quant_dynamic(v, ct)[1]
            assert d.shape[1] > 1 and (d[:, 1:] != d[:, :-1]).all() and (d[1:] != d[:-1]).all(), (family, ct)


# ==== GPU helpers ===========================================================================================================
def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@functools.lru_cache(maxsize=None)
def device_product(P):
    """The exact products on the device (float64), every entry's rows stacked; as numpy."""
    A = dev(P.a).double()
    out = torch.empty((P.rows, P.n), dtype=torch.float64, device="cuda")
    for e, lo, hi in P.entries():
        out[lo:hi] = A[lo:hi] @ dev(P.bt[e]).double().t()
    return out.cpu().numpy()


class Operands:
    """P's FP8 bytes of a pair on the device at padded pitches, the padding FP8 NaN: A (a batch's entries 32 bytes apart)
    and B^T (entries 48 bytes apart); a grouped call's offsets."""

    def __init__(self, P, pair):
        ta, tb = pair
        a8 = f8.encode(P.a, ta)
        if P.stack == "bat":
            a8 = a8.reshape(P.E, P.sizes[0], P.k)
        self.A, self.lda, self.stride_a = fg.padded(a8, fg.pad16(P.k) + 16, entry_gap=32 if P.stack == "bat" else 0)
        self.B, self.ldb, self.stride_b = fg.padded(f8.encode(P.bt, tb), fg.pad16(P.k) + 32, entry_gap=48)
        self.offs = torch.tensor([int(x) for x in P.starts[1:]], dtype=torch.int32, device="cuda")


def c_buffer(P, o):
    return torch.full((P.c_rows, P.ldc), float("nan"), dtype=f8.out_dtype(o), device="cuda")


def check_c(C, want_dev, what):
    """The whole C buffer, fences included, against want (placed, float32 on the device), bit for bit."""
    assert tr.same_bits(C.float(), want_dev), what


def check_schedule(gemm, P, name, bn, sms, what):
    assert gemm.last_kernel() == name, (what, gemm.last_kernel())
    assert bt.last_schedule(gemm) == schedule(P.stack, P.sizes, P.n, bn, sms), what
    assert reaches_all(P.stack, P.sizes, P.n, P.k, bn, sms), what


def set_width(hooks, mode):
    """set_bn for a mode; promoted and blockwise get a forced 256 that they must ignore.  Returns (accum, bn, fast)."""
    accum, bn = accum_of(mode)
    hooks.b200_gemm_debug_set_bn(bn if accum == "fast" else 256)
    return accum, bn or 128, int(accum == "fast")


def run_single(gemm, P, ops, pair, o, fast, Sa, Sb, bias):
    C = c_buffer(P, o)
    Bi = torch.from_numpy(bias).to(f8.out_dtype(o)).cuda() if bias is not None else None
    rc = gemm.lib.b200_gemm_fp8(f8.OP_N, f8.OP_T, *pair, P.sizes[0], P.n, P.k, ops.A.data_ptr(), ops.lda,
                                ops.B.data_ptr(), ops.ldb, Sa.data_ptr(), int(Sa.numel() > 1), Sb.data_ptr(),
                                int(Sb.numel() > 1), Bi.data_ptr() if Bi is not None else None, C.data_ptr(), P.ldc, o,
                                fast, None)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return C


# ==== b200_gemm_fp8: 36 kernels =============================================================================================
@gpu
def test_single_matrix_kernels(gemm, hooks, sms):
    """Every pair, C type and width of b200_gemm_fp8 (fast 256 / 192 / 128, promoted) at one multi-round, ring-wrapping
    shape with a ragged raster group: rowwise power-of-two scales and a bias, or tensorwise scales.  Then the fast 256 and
    promoted kernels at forced group rows 128, 384 and 640."""
    P = problem("single", sms)
    acc = device_product(P)
    ops = {pair: Operands(P, pair) for pair in PAIRS}
    scales = {"row": (dev(P.sa_pow2), dev(P.sb_pow2[0]), P.bias, P.sa_pow2, P.sb_pow2),
              "tensor": (dev(P.s_tensor[:1]), dev(P.s_tensor[1:]), None, np.full(P.rows, P.s_tensor[0], np.float32),
                         np.full((1, P.n), P.s_tensor[1], np.float32))}
    wants = {}

    def want(o, how):
        if (o, how) not in wants:
            _, _, bias, sa, sb = scales[how]
            wants[(o, how)] = dev(P.place(rowwise_want(P, acc, sa, sb, bias, o)))
        return wants[(o, how)]

    for pair, o, mode in SINGLE_CASES:
        how = rowwise_scaling(pair, o, mode)
        accum, bn, fast = set_width(hooks, mode)
        C = run_single(gemm, P, ops[pair], pair, o, fast, *scales[how][:3])
        what = (pair, OUT_NAME[o], mode, how)
        check_schedule(gemm, P, kernel_name(pair, o, accum, bn), bn, sms, what)
        check_c(C, want(o, how), what)
    pair, o = (E4M3, E4M3), OUT_BF16
    for mode in ("fast256", "promoted"):
        accum, bn, fast = set_width(hooks, mode)
        how = rowwise_scaling(pair, o, mode)
        for rows in RASTER_ROWS:
            hooks.b200_gemm_debug_set_group_rows(rows)
            C = run_single(gemm, P, ops[pair], pair, o, fast, *scales[how][:3])
            check_schedule(gemm, P, kernel_name(pair, o, accum, bn), bn, sms, (mode, rows))
            check_c(C, want(o, how), (mode, "group rows", rows))
        hooks.b200_gemm_debug_set_group_rows(0)


@gpu
def test_fp32_c_never_splits_k(gemm, hooks, sms):
    """A partial last round with a long K (where a 16-bit fp32-C kernel splits the tail 4 ways): the FP8 kernels run
    whole tiles, fast and promoted, and the promoted result is exact."""
    m, n, k = 384, 256, 8192
    assert ts.tc_split(m, n, k, "bf16", 128, sms) > 1
    rng = np.random.default_rng(5)
    a, b = rng.integers(-2, 3, (m, k)).astype(np.float32), rng.integers(-2, 3, (k, n)).astype(np.float32)
    A, Bt = dev(f8.encode(a, E4M3)), dev(f8.encode(np.ascontiguousarray(b.T), E4M3))
    one = torch.ones(1, device="cuda")
    hooks.b200_gemm_debug_set_bn(128)
    for fast in (1, 0):
        C = torch.full((m, n), float("nan"), device="cuda")
        assert gemm.lib.b200_gemm_fp8(f8.OP_N, f8.OP_T, E4M3, E4M3, m, n, k, A.data_ptr(), k, Bt.data_ptr(), k,
                                      one.data_ptr(), 0, one.data_ptr(), 0, None, C.data_ptr(), n, OUT_F32, fast,
                                      None) == 0
        torch.cuda.synchronize()
        assert bt.last_schedule(gemm) == schedule("none", [m], n, 128, sms) == (6, 1, 6, 6)
    assert torch.equal(C.double(), dev(a).double() @ dev(b).double())


# ==== b200_gemm_fp8_blockwise: 9 kernels ====================================================================================
def blk_scale_tensors(P, recipe, outer_a=False):
    """The recipe's scales on the device, NaN between their rows and k-blocks; outer_a: scale_a outer-dim-major (torch's
    layout, one matrix only)."""
    sa, sb = P.blk_scales(recipe)
    Sa = dev(np.ascontiguousarray(sa.T)).t() if outer_a else bfg.nan_padded(sa)
    return Sa, bfg.nan_padded(sb)


def run_blockwise(gemm, P, ops, pair, o, recipe, Sa, Sb, bias):
    C = c_buffer(P, o)
    Bi = torch.from_numpy(bias).to(f8.out_dtype(o)).cuda() if bias is not None else None
    rc = gemm.lib.b200_gemm_fp8_blockwise(f8.OP_N, f8.OP_T, *pair, P.sizes[0], P.n, P.k, ops.A.data_ptr(), ops.lda,
                                          ops.B.data_ptr(), ops.ldb, Sa.data_ptr(), recipe[0], *Sa.stride(),
                                          Sb.data_ptr(), recipe[1], *Sb.stride(),
                                          Bi.data_ptr() if Bi is not None else None, C.data_ptr(), P.ldc, o, None)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return C


@gpu
def test_single_matrix_blockwise_kernels(gemm, hooks, sms):
    """Every pair and C type of b200_gemm_fp8_blockwise, each recipe with random fp32 scales and a bias, scale_a row-major
    or outer-dim-major; then one kernel at forced group rows 128, 384 and 640."""
    P = problem("single_blk", sms)
    ops = {pair: Operands(P, pair) for pair in PAIRS}
    for i, (pair, o, recipe) in enumerate(BLK_CASES):
        if i % len(PAIRS) == 0:
            want = dev(P.place(blk_want(P, recipe, o, P.bias)))
        set_width(hooks, "blk")
        Sa, Sb = blk_scale_tensors(P, recipe, outer_a=PAIRS.index(pair) == 1)
        C = run_blockwise(gemm, P, ops[pair], pair, o, recipe, Sa, Sb, P.bias)
        what = (pair, OUT_NAME[o], recipe)
        check_schedule(gemm, P, kernel_name(pair, o, "blk", 128), 128, sms, what)
        check_c(C, want, what)
    for rows in RASTER_ROWS:                             # the last case's kernel and data
        hooks.b200_gemm_debug_set_group_rows(rows)
        C = run_blockwise(gemm, P, ops[pair], pair, o, recipe, Sa, Sb, P.bias)
        check_schedule(gemm, P, kernel_name(pair, o, "blk", 128), 128, sms, ("group rows", rows))
        check_c(C, want, ("group rows", rows))


# ==== b200_gemm_fp8_q8 / _blockwise_q8: 24 kernels ==========================================================================
SENTINEL8 = 0xA5


def run_q8(gemm, P, ops, pair, ct, accum, act, sr=None, dynamic=False, outer=False):
    """The FP8-output call into a sentinel-filled C (one row and 16 columns of fence) and scale_c (8 fence floats on each
    side; outer: outer-dim-major).  Returns the C buffer and the scale_c buffer (CUDA uint8 / int32)."""
    m, n = P.sizes[0], P.n
    qn = cdiv(n, 128)
    ldc = n + 16
    C = torch.full((m + 1, ldc), SENTINEL8, dtype=torch.uint8, device="cuda")
    S = torch.full((8 + m * qn + 8,), fo.SC_SENTINEL, dtype=torch.int32, device="cuda")
    sc_row, sc_blk = (1, m) if outer else (qn, 1)
    Sr = dev(np.float32([sr])) if sr is not None else None
    Bi = torch.from_numpy(P.bias).bfloat16().cuda()
    out = (ct, C.data_ptr(), ldc, Sr.data_ptr() if Sr is not None else None, S.data_ptr() + 4 * 8 if dynamic else None,
           sc_row, sc_blk, None)
    head = (f8.OP_N, f8.OP_T, *pair, m, n, P.k, ops.A.data_ptr(), ops.lda, ops.B.data_ptr(), ops.ldb)
    if accum == "blk":
        Sa, Sb = blk_scale_tensors(P, (1, 128))
        rc = gemm.lib.b200_gemm_fp8_blockwise_q8(*head, Sa.data_ptr(), 1, *Sa.stride(), Sb.data_ptr(), 128, *Sb.stride(),
                                                 Bi.data_ptr(), act, *out)
    else:
        Sa, Sb = dev(P.sa_rand), dev(P.sb_rand[0])
        rc = gemm.lib.b200_gemm_fp8_q8(*head, Sa.data_ptr(), 1, Sb.data_ptr(), 1, Bi.data_ptr(), act,
                                       int(accum == "fast"), *out)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return C, S


def q8_expected(P, v, ct, sr=None, dynamic=False, outer=False):
    """The whole C and scale_c buffers run_q8 must leave: the quantisation of v (test_fp8_out_gpu's quantisers) inside
    the fences."""
    m, n = v.shape
    qn = cdiv(n, 128)
    C = np.full((m + 1, n + 16), SENTINEL8, np.uint8)
    S = np.full(8 + m * qn + 8, fo.SC_SENTINEL, np.int32)
    if dynamic:
        C[:m, :n], d = fo.quant_dynamic(v, ct)
        S[8:8 + m * qn] = np.ascontiguousarray(d.T if outer else d).reshape(-1).view(np.int32)
    else:
        C[:m, :n] = fo.quant_static(v, ct, sr)
    return dev(C), dev(S)


@gpu
def test_fp8_output_kernels(gemm, hooks, sms):
    """Every pair, C type and input form of the FP8-output GEMMs (fast 256 / 128, promoted, blockwise) with bias and
    ReLU, in static mode (s_r) and dynamic mode (row-major or outer-dim-major scale_c): C and scale_c bit for bit,
    nothing written outside them, every scale written.  A forced 192 takes the heuristic's width; one kernel runs at
    forced group rows 128, 384 and 640; GELU in each mode through the device's own activation."""
    Ps = {"row": problem("single", sms), "blk": problem("single_blk", sms)}
    vs = {"row": q8_v(Ps["row"], device_product(Ps["row"])), "blk": q8_v(Ps["blk"])}
    ops = {(key, pair): Operands(Ps[key], pair) for key in Ps for pair in PAIRS}
    wants = {}

    def want(key, ct, dynamic, outer):
        if (key, ct, dynamic, outer) not in wants:
            wants[(key, ct, dynamic, outer)] = q8_expected(Ps[key], fo.relu_np(vs[key]), ct, Ps[key].s_r, dynamic, outer)
        return wants[(key, ct, dynamic, outer)]

    def case(pair, ct, mode, dynamic, outer=False, bn=None):
        key = "blk" if mode == "blk" else "row"
        P = Ps[key]
        accum, bn_model, _ = set_width(hooks, mode)
        if bn is not None:
            hooks.b200_gemm_debug_set_bn(bn)
            bn_model = fp8_width("none", P.sizes, P.n, sms, "fast", force=bn, fp8_out=True)
        C, S = run_q8(gemm, P, ops[(key, pair)], pair, ct, accum, fo.ACT_RELU, None if dynamic else P.s_r, dynamic, outer)
        what = (pair, fo.CT_NAME[ct], mode, "dynamic" if dynamic else "static", outer)
        check_schedule(gemm, P, kernel_name(pair, fo.CT_NAME[ct], accum, bn_model), bn_model, sms, what)
        wc, ws = want(key, ct, dynamic, outer)
        assert torch.equal(C, wc), what
        assert torch.equal(S, ws), what

    for i, (pair, ct, mode) in enumerate(Q8_CASES):
        case(pair, ct, mode, False)
        case(pair, ct, mode, True, outer=i % 2 == 1)
    case((E4M3, E4M3), E4M3, "fast256", True, bn=192)
    for rows in RASTER_ROWS:
        hooks.b200_gemm_debug_set_group_rows(rows)
        case((E4M3, E5M2), E5M2, "fast256", True)
    hooks.b200_gemm_debug_set_group_rows(0)
    # GELU: v = act(v) by the device's own epilogue; same bytes, or both zero (the oracle's beta step turns -0 into +0)
    P = Ps["row"]
    v = fo.act_dev(gemm, vs["row"], fo.ACT_GELU)
    set_width(hooks, "fast128")
    for dynamic in (False, True):
        C, S = run_q8(gemm, P, ops[("row", (E4M3, E4M3))], (E4M3, E4M3), E4M3, "fast", fo.ACT_GELU,
                      None if dynamic else P.s_r, dynamic)
        assert gemm.last_kernel() == kernel_name((E4M3, E4M3), "oe4m3", "fast", 128)
        wc, ws = q8_expected(P, v, E4M3, P.s_r, dynamic)
        assert fo.same_or_both_zero(C.cpu().numpy()[:-1, :P.n], wc.cpu().numpy()[:-1, :P.n], E4M3), dynamic
        assert torch.equal(C[:, P.n:], wc[:, P.n:]) and torch.equal(C[-1], wc[-1])
        assert torch.equal(S, ws), dynamic


# ==== grouped and batched, rowwise: 72 kernels ==============================================================================
def run_stacked(gemm, P, ops, pair, o, fast):
    C = c_buffer(P, o)
    if P.stack == "grp":
        Sa, Sb = dev(P.sa_pow2), bfg.nan_padded(P.sb_pow2)
        rc = gemm.lib.b200_gemm_fp8_grouped(*pair, P.rows, P.n, P.k, ops.A.data_ptr(), ops.lda, ops.B.data_ptr(), ops.ldb,
                                            ops.stride_b, ops.offs.data_ptr(), P.E, Sa.data_ptr(),
                                            Sb.data_ptr(), Sb.stride(0), C.data_ptr(), P.ldc, o, fast, None)
    else:
        Sa, Sb = bfg.nan_padded(P.sa_pow2.reshape(P.E, -1)), bfg.nan_padded(P.sb_pow2)
        rc = gemm.lib.b200_gemm_fp8_batched(*pair, P.sizes[0], P.n, P.k, ops.A.data_ptr(), ops.lda, ops.stride_a,
                                            ops.B.data_ptr(), ops.ldb, ops.stride_b, Sa.data_ptr(), Sa.stride(0),
                                            Sb.data_ptr(), Sb.stride(0), C.data_ptr(), P.ldc, P.stride_c, P.E, o, fast,
                                            None)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return C


@gpu
@pytest.mark.parametrize("stack", ["grp", "bat"])
def test_stacked_kernels(gemm, hooks, sms, stack):
    """Every pair, C type and width of b200_gemm_fp8_grouped / _batched (the groups: a 2157-row one, two empty, one of 1
    row) against the exact oracle, not only against per-group calls; rows after the last group, the gap row after each
    batch entry and the columns past n stay NaN.  Then the fast 256 kernel at forced group rows 128, 384 and 640."""
    P = problem(stack, sms)
    acc = device_product(P)
    ops = {pair: Operands(P, pair) for pair in PAIRS}
    wants = {o: dev(P.place(rowwise_want(P, acc, P.sa_pow2, P.sb_pow2, None, o))) for o in OUTS}
    for _, pair, o, mode in [c for c in STACK_CASES if c[0] == stack]:
        accum, bn, fast = set_width(hooks, mode)
        C = run_stacked(gemm, P, ops[pair], pair, o, fast)
        what = (pair, OUT_NAME[o], mode)
        check_schedule(gemm, P, kernel_name(pair, o, accum, bn, stack), bn, sms, what)
        check_c(C, wants[o], what)
    pair, o = (E5M2, E4M3), OUT_F16
    accum, bn, fast = set_width(hooks, "fast256")
    for rows in RASTER_ROWS:
        hooks.b200_gemm_debug_set_group_rows(rows)
        C = run_stacked(gemm, P, ops[pair], pair, o, fast)
        check_schedule(gemm, P, kernel_name(pair, o, accum, bn, stack), bn, sms, ("group rows", rows))
        check_c(C, wants[o], ("group rows", rows))


# ==== grouped and batched, blockwise: 18 kernels ============================================================================
def run_stacked_blk(gemm, P, ops, pair, o, recipe):
    C = c_buffer(P, o)
    Sa, Sb = blk_scale_tensors(P, recipe)
    if P.stack == "grp":
        rc = gemm.lib.b200_gemm_fp8_blockwise_grouped(*pair, P.rows, P.n, P.k, ops.A.data_ptr(), ops.lda,
                                                      ops.B.data_ptr(), ops.ldb, ops.stride_b, ops.offs.data_ptr(), P.E,
                                                      Sa.data_ptr(), *Sa.stride(), Sb.data_ptr(), recipe[1],
                                                      Sb.stride(1), Sb.stride(2), Sb.stride(0), C.data_ptr(), P.ldc, o,
                                                      None)
    else:
        rc = gemm.lib.b200_gemm_fp8_blockwise_batched(*pair, P.sizes[0], P.n, P.k, ops.A.data_ptr(), ops.lda,
                                                      ops.stride_a, ops.B.data_ptr(), ops.ldb, ops.stride_b,
                                                      Sa.data_ptr(), recipe[0], Sa.stride(1), Sa.stride(2), Sa.stride(0),
                                                      Sb.data_ptr(), recipe[1], Sb.stride(1), Sb.stride(2), Sb.stride(0),
                                                      C.data_ptr(), P.ldc, P.stride_c, P.E, o, None)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return C


@gpu
@pytest.mark.parametrize("stack", ["grp", "bat"])
def test_stacked_blockwise_kernels(gemm, hooks, sms, stack):
    """Every pair and C type of b200_gemm_fp8_blockwise_grouped / _batched, every recipe each accepts, random fp32 scales
    NaN-fenced between rows, k-blocks and entries, against the FMA-chain oracle bit for bit.  Then one kernel at forced
    group rows 128, 384 and 640."""
    P = problem(stack + "_blk", sms)
    ops = {pair: Operands(P, pair) for pair in PAIRS}
    for _, pair, o, recipe in [c for c in STACK_BLK_CASES if c[0] == stack]:
        if pair == PAIRS[0]:
            want = dev(P.place(blk_want(P, recipe, o)))
        set_width(hooks, "blk")
        C = run_stacked_blk(gemm, P, ops[pair], pair, o, recipe)
        what = (pair, OUT_NAME[o], recipe)
        check_schedule(gemm, P, kernel_name(pair, o, "blk", 128, stack), 128, sms, what)
        check_c(C, want, what)
    for rows in RASTER_ROWS:                             # the last case's kernel and data
        hooks.b200_gemm_debug_set_group_rows(rows)
        C = run_stacked_blk(gemm, P, ops[pair], pair, o, recipe)
        check_schedule(gemm, P, kernel_name(pair, o, "blk", 128, stack), 128, sms, ("group rows", rows))
        check_c(C, want, ("group rows", rows))
