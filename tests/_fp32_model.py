"""Exact models of the fp32 precision modes of b200_gemm_f32 (numpy, CPU only).

Each model restates the operand transform a mode applies before the tensor cores see the operands,
exactly as the kernels in csrc/gemm_tc.cuh implement it, and sums the plane products the kernel issues
in float64.  model(A, B, mode) answers: what would this mode return if its accumulation were exact?

  tf32    wgmma ignores the low 13 mantissa bits of each fp32 operand (truncation).
  bf16x3  split_planes_kernel: p1 = bf16_rne(x), p2 = bf16_rne(x - p1), p3 = bf16_rne(x - p1 - p2), the
          subtractions exact in fp32; a finite x whose first plane would round to inf gets +-0x7f7f (the
          residual stays exact), a non-finite x gives p1 = x and zero lower planes.  Products ProdX3.
  bf16x2  the first two of those planes, products ProdX2.
  f16x2   e = pow2_exp(row max of A / column max of B); x' = fp32(x * 2^-e) (the kernel may round an x' below
          2^-126 twice; such values split into zero planes either way); h1 = fp16_rne(x'),
          h2 = fp16_rne(x' - h1) (fp16 subnormals kept); products ProdX2 of the h planes; the sum is
          multiplied by 2^(e_row + e_col).

The float64 sum is exact for the known-answer operands of the tests (their products span fewer than
53 bits); elsewhere its rounding, below K * 2^-53 of the sum of |products|, is far under every bound the
tests use.  The mutation keywords of model() exist so that the tests can show that a wrong kernel
would change the expected bits."""
import numpy as np

F32_MAX = float(np.finfo(np.float32).max)
BF16_MAX = np.float32(np.uint32(0x7F7F0000).view(np.float32))

# (plane of A, plane of B) of every product the kernel issues, in issue order (gemm_tc.cuh ProdX3 / ProdX2)
PRODS = {"bf16x3": ((0, 2), (2, 0), (1, 1), (0, 1), (1, 0), (0, 0)),
         "bf16x2": ((0, 1), (1, 0), (0, 0)),
         "f16x2": ((0, 1), (1, 0), (0, 0)),
         "tf32": ((0, 0),)}
NPLANES = {"bf16x3": 3, "bf16x2": 2, "f16x2": 2, "tf32": 1}
MMA_K = {"bf16x3": 16, "bf16x2": 16, "f16x2": 16, "tf32": 8}


def f32(x):
    return np.asarray(x, dtype=np.float32)


def bits(x):
    return f32(x).view(np.uint32)


def from_bits(b):
    return np.asarray(b, dtype=np.uint32).view(np.float32)


# ---- operand transforms ---------------------------------------------------------------------------------
def tf32(x, rne=False):
    """The tf32 operand wgmma reads: the low 13 mantissa bits dropped (rne=True: rounded instead, a mutant)."""
    b = bits(x).astype(np.uint64)
    if rne:
        b = b + 0xFFF + ((b >> 13) & 1)
    r = from_bits(((b >> 13) << 13).astype(np.uint32))
    x = f32(x)
    return np.where(np.isfinite(x), r, x)


def bf16_round(x, trunc=False):
    """fp32 -> bf16 (as fp32), round to nearest even (cvt.rn.bf16x2.f32); NaN stays NaN.  trunc: chop (a mutant)."""
    b = bits(x).astype(np.uint64)
    if not trunc:
        b = b + 0x7FFF + ((b >> 16) & 1)
    r = from_bits(((b >> 16) << 16).astype(np.uint32))
    x = f32(x)
    return np.where(np.isnan(x), x, r)


def bf16_planes(x, n=3, trunc=False):
    """split_planes_kernel: n bf16 planes of x (each as fp32), with the range-edge rules of the kernel."""
    r = f32(x).copy()
    fin = np.isfinite(r)
    planes = []
    for _ in range(n):
        p = bf16_round(r, trunc)
        p = np.where(fin & np.isinf(p), np.copysign(BF16_MAX, r), p).astype(np.float32)
        planes.append(p)
        with np.errstate(invalid="ignore"):
            r = np.where(fin, r - p, np.float32(0)).astype(np.float32)
    return planes


def pow2_exp(maxv):
    """gemm_tc.cuh pow2_exp: e with maxv * 2^-e in [0.5, 1) for finite nonzero maxv (subnormals by their leading
    bit), 0 for zero, inf or NaN."""
    b = bits(maxv).astype(np.int64)
    ef = (b >> 23) & 0xFF
    mant = b & 0x7FFFFF
    lead = np.frexp(np.maximum(mant, 1).astype(np.float64))[1] - 1          # leading bit of a subnormal
    e = np.where(ef == 255, 0, np.where(ef != 0, ef - 126, np.where(mant == 0, 0, lead - 148)))
    return e.astype(np.int64)


def absmax(x, axis):
    """fmaxf reduction of |x| from 0 (NaN is skipped, as fmaxf does)."""
    with np.errstate(invalid="ignore"):
        m = np.nanmax(np.abs(f32(x)), axis=axis, initial=0.0)
    return f32(m)


def f16_planes(x, e, drop_h2=False, trunc=False):
    """split_f16x8 after the power-of-two scaling: x' = fp32(x * 2^-e) (one rounding), h1 = fp16(x'),
    h2 = fp16(x' - h1), each returned as float64.  trunc: fp16 rounding by chopping (a mutant)."""
    x = f32(x).astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        xs = f32(x * np.ldexp(1.0, -e))

        def to16(v):
            if not trunc:
                return v.astype(np.float16)
            h = v.astype(np.float16)                       # chop toward zero: step back where RNE went up
            up = np.abs(h.astype(np.float32)) > np.abs(v)
            hb = h.view(np.uint16).astype(np.int32) - up.astype(np.int32)
            return np.where(np.isfinite(v), hb.astype(np.uint16).view(np.float16), h)
        h1 = to16(xs)
        h2 = to16(f32(xs - h1.astype(np.float32)))
    if drop_h2:
        h2 = np.zeros_like(h2)
    return h1.astype(np.float64), h2.astype(np.float64)


def planes(A, B, mode, trunc=False, drop_h2=False, exp_shift=0):
    """(planes of A, planes of B, row exponents, column exponents), planes as float64."""
    if mode == "tf32":
        return [tf32(A, rne=trunc).astype(np.float64)], [tf32(B, rne=trunc).astype(np.float64)], 0, 0
    if mode in ("bf16x3", "bf16x2"):
        n = NPLANES[mode]
        return ([p.astype(np.float64) for p in bf16_planes(A, n, trunc)],
                [p.astype(np.float64) for p in bf16_planes(B, n, trunc)], 0, 0)
    ea = pow2_exp(absmax(A, 1)) + exp_shift
    eb = pow2_exp(absmax(B, 0)) + exp_shift
    pa = f16_planes(A, ea[:, None], drop_h2, trunc)
    pb = f16_planes(B, eb[None, :], drop_h2, trunc)
    return list(pa), list(pb), ea, eb


def model(A, B, mode, prods=None, trunc=False, drop_h2=False, exp_shift=0, unscale_shift=0, absolute=False):
    """What `mode` returns for A (m x k) * B (k x n) if its accumulation were exact, float64 m x n.

    Mutants: prods (another product list), trunc (chopped instead of rounded splits; for tf32 the other way
    round), drop_h2 (F16X2 without its second plane), exp_shift (the F16X2 pre-pass scales rows and columns with
    exponents off by that much, the epilogue does not), unscale_shift (only the epilogue's exponent off).
    absolute=True: the sum of |plane products| instead, in the same units (for error bounds)."""
    pa, pb, ea, eb = planes(A, B, mode, trunc, drop_h2, exp_shift)
    prods = PRODS[mode] if prods is None else prods
    m, n = f32(A).shape[0], f32(B).shape[1]
    acc = np.zeros((m, n))
    with np.errstate(invalid="ignore", over="ignore"):
        for i, j in prods:
            acc = acc + (np.abs(pa[i]) @ np.abs(pb[j]) if absolute else pa[i] @ pb[j])
        if mode == "f16x2":
            e = ea[:, None] + eb[None, :] - 2 * exp_shift + unscale_shift
            acc = acc * np.ldexp(1.0, e.astype(np.int64))
    return acc


def accumulation_bound(A, B, mode, chunk, parts=1):
    """Bound on |GPU - model| from the fp32 accumulation alone.

    The kernel accumulates each chunk of `chunk` k-values in a fresh wgmma accumulator and adds chunks to a
    running sum with a rounded fp32 add; K-split parts are folded into C with rounded adds.  Assume each wgmma
    step (MMA_K products of each of the P plane products) adds its terms with at most 2 ulp of error relative
    to the sum of |terms| accumulated so far (the tensor core aligns to the largest addend and chops):
        steps per chunk = P * ceil(min(chunk, K) / MMA_K),  error <= steps * 2^-22 * S
    plus one half ulp per chunk fold, per part fold and for the final value: (chunks + parts + 1) * 2^-24 * S,
    where S is the sum of |plane products| (in the accumulator's units, then unscaled).  Accumulators of the
    bf16 / tf32 modes can reach the subnormal range: each step may also lose 2^-149 absolutely.  F16X2
    accumulators are multiples of 2^-48 (products of fp16 values), so they never do, but the unscaled result
    and every part fold may round to the fp32 subnormal grid: (parts + 1) * 2^-149."""
    k = f32(A).shape[1]
    P = len(PRODS[mode])
    kc = min(chunk, k) if chunk else k
    chunks = -(-k // kc)
    steps = P * -(-kc // MMA_K[mode])
    S = model(A, B, mode, absolute=True)
    rel = steps * 2.0 ** -22 + (chunks + parts + 1) * 2.0 ** -24
    absolute = (parts + 1 if mode == "f16x2" else P * chunks * -(-kc // MMA_K[mode])) * 2.0 ** -149
    return rel * S + absolute


def class_bound(A, B, mode):
    """Each mode's documented error class, |model - exact| <= bound (float64 m x n).  Derivations:

    bf16x3  x = p1 + p2 + p3 exactly while the planes are normal bf16 (three RNE chunks of 8 bits cover 24 bits);
            the dropped products a2b3 + a3b2 + a3b3 are below (2 * 2^-8 * 2^-16 + 2^-32) |a||b| < 2^-22 |a||b|:
            elementwise 2^-22 (|A||B|)ij.
    bf16x2  x - p1 - p2 is below 2^-16 |x|; with the dropped a2b2 (<= 2^-16 |a||b|) the error per term is below
            3.1 * 2^-16 |a||b|: elementwise 2^-14 (|A||B|)ij.
    tf32    chopping 13 of 23 mantissa bits leaves a relative error below 2^-10 per operand:
            elementwise 2^-9 (|A||B|)ij.
    f16x2   |x'| < 1 after scaling; h1 + h2 misses x' by at most 2^-24 (half the quantum of h2, whose smallest is
            the fp16 subnormal 2^-24); per term |a'b' - kept| <= 2^-24 + 2^-24 + 2^-24 (the dropped h2 h2) + 2^-48,
            unscaled by 2^(e_row + e_col) <= 4 rowmax colmax: normwise 2^-20 K rowmax_i colmax_j.
    Exception (bf16 / tf32 modes): where an operand is below 2^-110 its lower planes fall under the normal bf16 /
    tf32 range and the split loses bits absolutely: |x - planes| <= 2^-134 (half the bf16 subnormal quantum
    2^-133; tf32 chops to 2^-136).  That adds 2^-133 (sum_k |B(k,j)| + sum_k |A(i,k)|)."""
    A64, B64 = np.abs(f32(A).astype(np.float64)), np.abs(f32(B).astype(np.float64))
    if mode == "f16x2":
        k = A64.shape[1]
        ra, cb = absmax(A, 1).astype(np.float64), absmax(B, 0).astype(np.float64)
        return 2.0 ** -20 * k * ra[:, None] * cb[None, :]
    rel = {"bf16x3": 2.0 ** -22, "bf16x2": 2.0 ** -14, "tf32": 2.0 ** -9}[mode]
    return rel * (A64 @ B64) + 2.0 ** -133 * (A64.sum(1)[:, None] + B64.sum(0)[None, :])
