"""The per-device state the library carries from one call to the next, across streams, host threads and back-to-back
calls without a synchronise: the K-split flag slots, the split workspace, the double-buffered F16X2 column maxima,
the auxiliary pre-pass stream, the tensor-map cache and PDL launches that rely on griddepcontrol.wait.

Every case takes the path it names: shapes come from the schedule model of test_tile_schedules_gpu.py, and the
split that b200_gemm_debug_last_schedule reports is asserted after each tensor-core call.  References are exact, so a
reordered fold or a stale value changes bits:
  - 16-bit operands are small dyadic numbers (every partial sum exact in fp32), with beta = 0 and beta = 0.5 on a
    pre-filled C (part 0 alone applies beta, so a part that folds before part 0 has stored changes the result);
  - the fp32 modes use the known-answer operands of test_fp32_range_gpu.py and the exact model of _fp32_model.py;
  - int8 uses the CPU oracle.
The shape predictions, the exactness margins and the sensitivity of the model to a stale maximum need no GPU."""
import ctypes as C
import threading

import numpy as np
import pytest

import _fp32_model as fm
import _libs
import test_tile_schedules_gpu as ts
from test_fp32_range_gpu import exact_accumulation_margin, ka_operands

try:
    import torch
except ImportError:          # the CPU tests need no torch
    torch = None

_NO_GPU = torch is None or not torch.cuda.is_available()


def gpu(test):
    """Marked gpu, and skipped where no CUDA device is visible."""
    return pytest.mark.gpu(pytest.mark.skipif(_NO_GPU, reason="needs a CUDA device")(test))


OP_N, OP_T = 0, 1
OUT_F32, OUT_BF16 = 0, 1
F32_STRICT, F32_TF32, F32_F16X2 = 0, 1, 5
BN = 128                     # every tensor-core case forces the 128-wide tile, so one model covers all kinds
SMS = (132, 114)             # H100 SXM and PCIe
LAYS = {"nn": (OP_N, OP_N), "nt": (OP_N, OP_T), "tn": (OP_T, OP_N), "tt": (OP_T, OP_T)}
cdiv = ts.cdiv


# ==== shapes and their schedules (no GPU) ===========================================================================
def short16(split, sms):
    """A few tiles whose tail takes `split` parts at BN = 128 (test_tile_schedules_gpu.split_case at bf16's K)."""
    m, n, k, _ = ts.split_case("bf16", split, sms, False)
    return m, n, k


BATCHED = (3, 100, 104, 1064)                 # batch, m, n, k: 3 tiles, 17 k-blocks -> 2 parts
TF32_NT = (128, 128, 520)                     # one tile, 17 k-blocks of 32 -> 2 parts (KA_SHAPES["split_tail"])
LONG_K = (120, 120, 1 << 22)                  # one tile cut into 4 parts of 2^20 K each: milliseconds on one stream


def s8_shape(sms):
    m, n, k, _ = ts.split_case("s8", 2, sms, False)
    return m, n, k


def schedule(m, n, k, kind, sms, batch=1):
    """(tiles, split) at BN = 128; a batch counts the tiles of every entry."""
    tiles = cdiv(m, ts.TILE_M) * cdiv(n, BN) * batch
    return tiles, ts.tc_split(cdiv(m, ts.TILE_M) * batch * ts.TILE_M, n, k, kind, BN, sms)


@pytest.mark.parametrize("sms", SMS)
def test_every_case_takes_a_split_tail(sms):
    for split in (2, 3, 4):
        m, n, k = short16(split, sms)
        assert ts.pick_bn(m, n, sms, "bf16", force=BN) == BN
        assert schedule(m, n, k, "bf16", sms)[1] == split
    b, m, n, k = BATCHED
    assert schedule(m, n, k, "bf16", sms, b) == (3, 2)
    assert schedule(*TF32_NT, "tf32", sms) == (1, 2)
    assert schedule(*s8_shape(sms), "s8", sms)[1] == 2
    assert schedule(*LONG_K, "bf16", sms) == (1, 4)
    assert schedule(256, 256, 1024, "bf16", sms)[1] == 2                 # the chain's bf16 -> fp32 step
    assert schedule(256, 256, 2048, "s8", sms)[1] == 2                   # the chain's int8 -> int32 step
    # bf16 C never takes the tail, so the chain's 16-bit-C steps need no flag slot
    assert ts.tc_split(256, 1024, 192, "bf16_obf16", BN, sms) == 1


def dyadic(shape, seed, lo=-8, hi=8, den=8.0, density=1.0):
    """Integers in [lo, hi] / den, zero with probability 1 - density (float64 numpy)."""
    rng = np.random.default_rng(seed)
    x = rng.integers(lo, hi + 1, shape) / den
    return x * (rng.random(shape) < density)


def c0_of(m, n, seed):
    return np.random.default_rng(seed).integers(-64, 65, (m, n)) * 2.0 ** -6


def tf32_case(seed, beta):
    m, n, k = TF32_NT
    A, B = ka_operands("tf32", m, n, k, seed)
    c0 = fm.f32(np.random.default_rng(seed).integers(-64, 65, (m, n)) * 2.0 ** -10)
    want = fm.model(A, B, "tf32") + beta * c0.astype(np.float64)
    return A, B, c0, want


@pytest.mark.parametrize("beta", [0.0, 0.5])
def test_tf32_known_answers_are_exact(beta):
    for seed in range(2000, 2016):
        A, B, c0, want = tf32_case(seed, beta)
        assert exact_accumulation_margin(A, B, "tf32", 1.0, c0, beta).min() > 1.0, seed
        assert (fm.f32(want).astype(np.float64) == want).all()


# ---- F16X2 sequence: the maxima of one call must never reach the next --------------------------------------------
# (layout, m, n, k).  op_b = N keeps B's column maxima in the double-buffered cmax, op_a = T keeps A^T's in amax; each
# call re-zeroes the idle half for the next one.  Steps 2 (amax) and 3 and 8 (cmax) clear a half wider than their own
# pre-pass covers, with the separate memset; step 5 grows cmax past any width used before (16384 to start, doubled on
# growth) while the earlier calls are still queued; step 4 interleaves pack_a / pack_b.
F16X2_STEPS = [("nn", 64, 3000, 256), ("tt", 3000, 96, 256), ("tn", 64, 3000, 256), ("nn", 64, 80, 256),
               ("packed", 64, 80, 256), ("tn", 64, 66000, 256), ("nt", 80, 80, 256), ("tt", 80, 80, 256),
               ("nn", 64, 80, 256)]
F16X2_STEP_EXP = 12          # each call's maxima operands are 2^12 smaller than the previous call's


def f16x2_step(i):
    """Known-answer A, B of step i (float32 numpy), scaled so that the operands whose maxima are kept in the shared
    buffers shrink by 2^12 per step, from 2^48; the other operand grows by as much, keeping the product near 1."""
    lay, m, n, k = F16X2_STEPS[i]
    A, B = ka_operands("f16x2", m, n, k, 3000 + i)
    down = 48 - F16X2_STEP_EXP * i
    ea, eb = {"nn": (-down, down), "tt": (down, -down), "tn": (down, down), "nt": (down, -down),
              "packed": (0, 0)}[lay]
    return fm.f32(np.ldexp(A.astype(np.float64), ea)), fm.f32(np.ldexp(B.astype(np.float64), eb))


def test_f16x2_sequence_model_sees_a_stale_maximum():
    """Every step is exact under the model, and the model with that step's exponents raised to the previous step's
    gives other bits: a maximum left over from the call before would show."""
    for i in range(len(F16X2_STEPS)):
        A, B = f16x2_step(i)
        assert np.isfinite(A).all() and np.isfinite(B).all()
        assert exact_accumulation_margin(A, B, "f16x2").min() > 1.0, i
        want = fm.model(A, B, "f16x2")
        assert (fm.f32(want).astype(np.float64) == want).all(), i
        assert np.count_nonzero(want) > want.size // 2
        stale = fm.f32(fm.model(A, B, "f16x2", exp_shift=F16X2_STEP_EXP))
        assert not np.array_equal(fm.bits(stale), fm.bits(fm.f32(want))), i


def test_argument_checks_come_before_the_device(gemm):
    """The entry points driven below refuse malformed calls before touching any device state."""
    lib = gemm.lib
    buf = (C.c_float * 256)()
    assert lib.b200_gemm_bf16_ex(2, OP_N, 4, 4, 4, 1.0, buf, 4, buf, 4, 0.0, buf, 4, OUT_F32, None) == -1
    assert lib.b200_gemm_f16_ex(OP_N, OP_N, 4, 4, 4, 1.0, buf, 3, buf, 4, 0.5, buf, 4, OUT_F32, None) == -1
    assert lib.b200_gemm_bf16_batched(OP_N, OP_N, 4, 4, 4, 1.0, buf, 4, -1, buf, 4, 16, 0.0, buf, 4, 16, 2, OUT_F32,
                                      None) == -1
    assert lib.b200_gemm_f32_op(OP_N, OP_T, 4, 4, 4, 1.0, buf, 4, buf, 3, 0.0, buf, 4, F32_TF32, None) == -1
    assert lib.b200_gemm_s8s32_op(OP_N, -1, 4, 4, 4, buf, 4, buf, 4, buf, 4, None) == -1
    assert lib.b200_gemm_bf16_grouped(OP_N, 8, 4, 4, 1.0, buf, 4, buf, 4, 16, None, 2, 0.0, buf, 4, OUT_F32, None) == -1


# ==== GPU helpers ===================================================================================================
@pytest.fixture
def hooks(gemm):
    """The hooks these tests set, back at their defaults afterwards whatever the outcome."""
    lib = gemm.lib
    try:
        yield lib
    finally:
        lib.b200_gemm_debug_set_bn(0)
        lib.b200_gemm_debug_set_split_tail(1)
        lib.b200_gemm_debug_set_pdl(1)
        lib.b200_gemm_debug_set_split_chunk(-1, -1)


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def last_schedule(lib):
    v = [C.c_int(-1) for _ in range(4)]
    lib.b200_gemm_debug_last_schedule(*[C.byref(x) for x in v])
    return tuple(x.value for x in v)


def cur():
    return torch.cuda.current_stream().cuda_stream


def dev(x, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    return t if dtype is None else t.to(dtype)


def stored(X, op):
    """Device tensor X (logical rows x cols) stored as op requires (X^T for OP_T) with a 16-element pitch: (view, ld)."""
    S = X.t() if op == OP_T else X
    r, c = S.shape
    buf = torch.zeros((r, ts.pitch(c)), dtype=X.dtype, device="cuda")
    buf[:, :c] = S
    return buf[:, :c], buf.stride(0)


def nan_c(m, n, c0=None, dtype=None):
    """C with an odd pitch, NaN (or 77) everywhere, c0 in the first n columns."""
    dtype = dtype or torch.float32
    buf = torch.empty((m, n + 1 + n % 2), dtype=dtype, device="cuda")
    buf.fill_(float("nan") if dtype.is_floating_point else 77)
    if c0 is not None:
        buf[:, :n] = c0
    return buf


def bits(t):
    t = t.contiguous()
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def same_bits(x, y):
    return x.shape == y.shape and torch.equal(bits(x.cpu()), bits(y.cpu()))


class Job:
    """One split-tail library call: issue(stream) queues it; after a synchronise, out[:, :n] must equal want bit for
    bit.  name / sched: the kernel and (tiles, split) the call must report."""

    def __init__(self, issue, out, n, want, name, sched, keep):
        self.issue, self.out, self.n, self.want, self.name, self.sched, self.keep = issue, out, n, want, name, sched, keep

    def run(self, lib, stream):
        rc = self.issue(stream)
        assert rc == 0, (self.name, rc)
        return lib.b200_gemm_last_kernel().decode(), last_schedule(lib)[:2]

    def got(self):
        return self.out[..., :self.n] if self.out.dim() == 2 else self.out

    def check(self, what=""):
        assert same_bits(self.got(), self.want), (self.name, what)


def job16(lib, kind, lay, split, sms, seed, beta):
    """bf16 / fp16 _ex with fp32 C in layout lay, alpha 1 or 2, beta 0 or 0.5 on a pre-filled C."""
    m, n, k = short16(split, sms)
    alpha = 2.0 if seed % 2 else 1.0
    A, B, c0 = dyadic((m, k), seed), dyadic((k, n), seed + 1), c0_of(m, n, seed + 2)
    want = fm.f32(alpha * (A @ B) + beta * c0)
    dt = torch.bfloat16 if kind == "bf16" else torch.float16
    op_a, op_b = LAYS[lay]
    Av, lda = stored(dev(A, dt), op_a)
    Bv, ldb = stored(dev(B, dt), op_b)
    out = nan_c(m, n, dev(fm.f32(c0)) if beta else None)
    fn = lib.b200_gemm_bf16_ex if kind == "bf16" else lib.b200_gemm_f16_ex
    issue = lambda st: fn(op_a, op_b, m, n, k, alpha, Av.data_ptr(), lda, Bv.data_ptr(), ldb, beta, out.data_ptr(),
                          out.stride(0), OUT_F32, st)
    name = f"tc_{'bf16' if kind == 'bf16' else 'f16'}{'' if lay == 'nn' else '_' + lay}_128x128"
    return Job(issue, out, n, torch.from_numpy(want), name, schedule(m, n, k, "bf16", sms), (Av, Bv))


def job_batched(lib, kind, sms, seed, beta):
    b, m, n, k = BATCHED
    A, B, c0 = dyadic((b, m, k), seed), dyadic((b, k, n), seed + 1), c0_of(b * m, n, seed + 2).reshape(b, m, n)
    want = fm.f32(A @ B + beta * c0)
    dt = torch.bfloat16 if kind == "bf16" else torch.float16
    Ad, Bd = dev(A, dt), dev(B, dt)
    out = dev(fm.f32(c0)) if beta else torch.full((b, m, n), float("nan"), device="cuda")
    fn = lib.b200_gemm_bf16_batched if kind == "bf16" else lib.b200_gemm_f16_batched
    issue = lambda st: fn(OP_N, OP_N, m, n, k, 1.0, Ad.data_ptr(), k, m * k, Bd.data_ptr(), n, k * n, beta,
                          out.data_ptr(), n, m * n, b, OUT_F32, st)
    name = f"tc_{'bf16' if kind == 'bf16' else 'f16'}_bat_128x128"
    return Job(issue, out, n, torch.from_numpy(want), name, schedule(m, n, k, "bf16", sms, b), (Ad, Bd))


def job_tf32_nt(lib, sms, seed, beta):
    """TF32 with B given as B^T: read in place, no workspace, so nothing but the flag slot orders it."""
    m, n, k = TF32_NT
    A, B, c0, want = tf32_case(seed, beta)
    Ad, Btd = dev(A), dev(np.ascontiguousarray(B.T))
    out = nan_c(m, n, dev(c0) if beta else None)
    issue = lambda st: lib.b200_gemm_f32_op(OP_N, OP_T, m, n, k, 1.0, Ad.data_ptr(), k, Btd.data_ptr(), k, beta,
                                            out.data_ptr(), out.stride(0), F32_TF32, st)
    return Job(issue, out, n, torch.from_numpy(fm.f32(want)), "tc_tf32_128x128", schedule(m, n, k, "tf32", sms),
               (Ad, Btd))


def job_s8_nt(lib, oracle, sms, seed):
    m, n, k = s8_shape(sms)
    a, b = _libs.gen_s8(oracle, m, k, seed), _libs.gen_s8(oracle, k, n, seed + 1)
    want = _libs.ref_s8(oracle, a, b)
    Ad, Btd = dev(a), dev(np.ascontiguousarray(b.T))
    out = nan_c(m, n, dtype=torch.int32)
    issue = lambda st: lib.b200_gemm_s8s32_op(OP_N, OP_T, m, n, k, Ad.data_ptr(), k, Btd.data_ptr(), k, out.data_ptr(),
                                              out.stride(0), st)
    return Job(issue, out, n, torch.from_numpy(want), "tc_s8_128x128", schedule(m, n, k, "s8", sms), (Ad, Btd))


def short_jobs(lib, oracle, sms, seed, split=2, kinds16=("bf16", "f16"), lays=tuple(LAYS)):
    """One of each short split call: 16-bit _ex in the given layouts, batched, TF32 NT and int8 NT."""
    jobs = []
    for kind in kinds16:
        for j, lay in enumerate(lays):
            jobs.append(job16(lib, kind, lay, split, sms, seed + 10 * len(jobs), 0.5 if j % 2 else 0.0))
        jobs.append(job_batched(lib, kind, sms, seed + 10 * len(jobs), 0.5 if seed % 2 else 0.0))
    jobs.append(job_tf32_nt(lib, sms, 2000 + (seed // 10) % 16, 0.5 if seed % 2 else 0.0))
    jobs.append(job_s8_nt(lib, oracle, sms, seed + 10 * len(jobs)))
    return jobs


def long_job(lib, sms):
    """bf16 -> fp32 C, beta = 0.5, one tile cut into 4 parts of 2^20 K: entries in {-1, 0, 1}, so every partial sum
    is an integer below 2^22 and exact."""
    m, n, k = LONG_K
    g = torch.Generator(device="cuda").manual_seed(77)
    A = torch.randint(-1, 2, (m, k), device="cuda", generator=g, dtype=torch.int8)
    B = torch.randint(-1, 2, (k, n), device="cuda", generator=g, dtype=torch.int8)
    c0 = torch.randint(-64, 65, (m, n), device="cuda", generator=g).float()
    ref = torch.zeros((m, n), dtype=torch.float64, device="cuda")
    for k0 in range(0, k, 1 << 18):
        ref += A[:, k0:k0 + (1 << 18)].double() @ B[k0:k0 + (1 << 18)].double()
    want = (ref + 0.5 * c0.double()).float()
    assert torch.equal(want.double(), ref + 0.5 * c0.double())
    Ab, Bb = A.bfloat16(), B.bfloat16()
    del A, B, ref
    out = nan_c(m, n, c0)
    issue = lambda st: lib.b200_gemm_bf16_ex(OP_N, OP_N, m, n, k, 1.0, Ab.data_ptr(), k, Bb.data_ptr(), n, 0.5,
                                             out.data_ptr(), out.stride(0), OUT_F32, st)
    return Job(issue, out, n, want.cpu(), "tc_bf16_128x128", schedule(m, n, k, "bf16", sms), (Ab, Bb))


def forked(*streams):
    """Side streams ordered after everything queued so far (operand uploads included)."""
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())


def joined(*streams):
    for s in streams:
        torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()


# ==== a. flag slots across streams ==================================================================================
@gpu
def test_flag_slots_across_streams(gemm, oracle, hooks, sms):
    """One long-K split call on S1 while S2 and S3 queue 24 short split calls each (bf16 and fp16 _ex in every layout,
    batched, TF32 NT, int8 NT), no host synchronise in between: each slot comes back many times while S1's launch
    still runs, and every result must be its exact answer."""
    lib = hooks
    lib.b200_gemm_debug_set_bn(BN)
    long = long_job(lib, sms)
    side = [short_jobs(lib, oracle, sms, 100 + 1000 * s) + short_jobs(lib, oracle, sms, 101 + 1000 * s) for s in (0, 1)]
    assert all(len(js) >= 20 for js in side)
    torch.cuda.synchronize()
    s1, s2, s3 = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    forked(s1, s2, s3)
    assert long.run(lib, s1.cuda_stream) == (long.name, long.sched)
    for a, b in zip(*side):
        for job, s in ((a, s2), (b, s3)):
            assert job.run(lib, s.cuda_stream) == (job.name, job.sched)
            assert job.sched[1] > 1
    joined(s1, s2, s3)
    long.check("long K on S1")
    for s, js in enumerate(side):
        for i, job in enumerate(js):
            job.check(("stream", s + 2, "call", i))


# ==== b. host threads ===============================================================================================
@gpu
def test_split_calls_from_two_host_threads(gemm, oracle, hooks, sms):
    """Two fresh host threads on one device, each on its own stream, 40 split calls each (ctypes drops the GIL, so the
    calls overlap on the host): every result exact, and each thread's last kernel and last schedule are its own.  The
    threads make no CUDA call of their own, so their first call must bind the device's context itself."""
    lib = hooks
    lib.b200_gemm_debug_set_bn(BN)
    plans = [short_jobs(lib, oracle, sms, 5000 + 10 * r, 2, ("bf16",), ("nn", "tt")) for r in range(8)], \
            [short_jobs(lib, oracle, sms, 7000 + 10 * r, 3, ("f16",), ("nt", "tn")) for r in range(8)]
    plans = [[j for js in p for j in js] for p in plans]
    assert all(len(p) >= 30 for p in plans)
    torch.cuda.synchronize()
    streams = (torch.cuda.Stream(), torch.cuda.Stream())
    forked(*streams)
    seen, errors = ([], []), []
    barrier = threading.Barrier(2)

    def worker(t):
        try:
            barrier.wait()
            for job in plans[t]:
                seen[t].append(job.run(lib, streams[t].cuda_stream))
        except BaseException as e:            # reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    joined(*streams)
    for t in range(2):
        assert seen[t] == [(j.name, j.sched) for j in plans[t]], t
        assert all(s[1] > 1 for _, s in seen[t])
        for i, job in enumerate(plans[t]):
            job.check(("thread", t, "call", i))


# ==== c. F16X2 maxima over a sequence on one stream =================================================================
@gpu
def test_f16x2_maxima_over_a_sequence(gemm, hooks):
    """F16X2 calls back to back on one stream, no synchronise: n shrinking from thousands to 80 (the separate clear
    of the idle half), growing past 65536 (cmax regrown while work is queued), NN / TT / TN / NT alternating (cmax and
    amax both rotate), pack_a / pack_b interleaved.  Each call's maxima operands are 2^12 smaller than the previous
    call's, so a maximum left over changes its bits; every result must equal the model."""
    steps = []
    for i, (lay, m, n, k) in enumerate(F16X2_STEPS):
        A, B = f16x2_step(i)
        steps.append((lay, dev(A), dev(B), fm.f32(fm.model(A, B, "f16x2"))))
    outs = [torch.full((s[1].shape[0], s[2].shape[1]), float("nan"), device="cuda") for s in steps]
    extra = torch.full_like(outs[4], float("nan"))
    views = []
    for lay, A, B, _ in steps:                 # the stored operands, uploaded before the sequence starts
        if lay == "packed":
            views.append((A, B))
            continue
        op_a, op_b = LAYS[lay]
        views.append((A.t().contiguous().t() if op_a else A, B.t().contiguous().t() if op_b else B))
    torch.cuda.synchronize()
    handles = []
    for i, ((lay, _, _, _), (Av, Bv), out) in enumerate(zip(steps, views, outs)):
        if lay == "packed":
            pa, pb = gemm.PackedA(Av, F32_F16X2), gemm.PackedB(Bv, F32_F16X2)
            handles += [pa, pb]
            gemm.gemm_f32_packed_ab(pa, pb, out)
            gemm.gemm_f32_packed(Av, pb, out=extra)
            assert gemm.last_kernel() == "tc_f16x2_128x128"
            continue
        assert gemm.operand_layout(tuple(Av.shape), Av.stride())[0] == LAYS[lay][0]
        gemm.gemm(Av, Bv, out, mode=F32_F16X2)
        assert gemm.last_kernel() == f"tc_f16x2{'' if lay == 'nn' else '_' + lay}_128x128", i
    torch.cuda.synchronize()
    for h in handles:
        h.close()
    for i, ((lay, _, _, want), out) in enumerate(zip(steps, outs)):
        got = out.cpu().numpy()
        bad = fm.bits(got) != fm.bits(want)
        assert not bad.any(), (i, lay, int(bad.sum()))
    assert np.array_equal(fm.bits(extra.cpu().numpy()), fm.bits(steps[4][3]))


# ==== d. dependent chains ===========================================================================================
GROUP_ROWS = (50, 0, 131, 60)            # rows of the chain's grouped call: the last 15 rows of C stay unwritten


def chain_inputs(oracle):
    """Inputs of one dependent chain, all uploaded up front (the chain itself only launches)."""
    d = {}
    m, k0, n = 256, 192, 1024
    d["A0"] = dev(dyadic((m, k0), 1, -1, 1, 1.0), torch.bfloat16)
    d["B0"] = dev(dyadic((k0, n), 2, -1, 1, 1.0), torch.bfloat16)
    d["B0b"] = dev(dyadic((k0, n), 3, -1, 1, 1.0), torch.bfloat16)
    d["B1"] = dev(dyadic((n, n), 4, -1, 1, 1.0, 1 / 32), torch.bfloat16)
    d["B2"] = dev(dyadic((n, 256), 5, -1, 1, 1.0, 1 / 32), torch.bfloat16)
    d["W"] = dev(fm.f32(dyadic((256, 200), 6)))
    d["W2"] = dev(fm.f32(dyadic((256, 136), 7)))
    d["W3"] = dev(fm.f32(dyadic((96, 136), 8)))
    d["Wg"] = dev(dyadic((4, n, 64), 9, -1, 1, 1.0, 1 / 32), torch.bfloat16)
    d["counts"] = dev(np.array(GROUP_ROWS, np.int32))
    a8, b8, b8b = _libs.gen_s8(oracle, 256, 512, 10), _libs.gen_s8(oracle, 512, 2048, 11), _libs.gen_s8(oracle, 2048, 256, 12)
    rng = np.random.default_rng(13)
    scales = fm.f32(rng.uniform(0.5, 2.0, 256) * 300.0 / (127.0 ** 2 * 512 ** 0.5))
    bias8 = fm.f32(rng.uniform(-20, 20, 256))
    q = _libs.requant_s8(oracle, _libs.ref_s8(oracle, a8, b8), scales, bias8)
    d["s8"] = (dev(a8), dev(b8), dev(b8b), dev(scales), dev(bias8))
    d["s8_want"] = (torch.from_numpy(q), torch.from_numpy(_libs.ref_s8(oracle, q, b8b)))
    return d


def run_chain(gemm, d, sync):
    """Each call reads what the previous one wrote; sync: a device synchronise after every step."""
    lib, st = gemm.lib, cur()
    o = {}
    step = torch.cuda.synchronize if sync else (lambda: None)
    m, n = 256, 1024

    def bf16_out(A, B, out, beta=0.0, bias=None, act=0):
        k = A.shape[1]
        rc = lib.b200_gemm_bf16_epi(OP_N, OP_N, A.shape[0], B.shape[1], k, 1.0, A.data_ptr(), A.stride(0),
                                    B.data_ptr(), B.stride(0), beta, out.data_ptr(), out.stride(0), OUT_BF16,
                                    bias.data_ptr() if bias is not None else None, act, st)
        assert rc == 0
        step()
    o["H"] = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
    bf16_out(d["A0"], d["B0"], o["H"])
    o["E"] = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
    bf16_out(d["A0"], d["B0b"], o["E"])
    o["bias"] = (o["H"][1] + o["E"][2]).contiguous()                                   # a torch kernel's output
    o["E0"] = o["E"].clone()
    step()
    bf16_out(o["H"], d["B1"], o["E"], beta=0.5, bias=o["bias"], act=gemm.ACT_RELU)     # bf16 C as beta * C, in place
    o["X"] = torch.full((m, 256), float("nan"), device="cuda")
    assert lib.b200_gemm_bf16_ex(OP_N, OP_N, m, 256, n, 1.0, o["E"].data_ptr(), n, d["B2"].data_ptr(), 256, 0.0,
                                 o["X"].data_ptr(), 256, OUT_F32, st) == 0              # bf16 C as the next operand
    o["X_split"] = last_schedule(lib)[1]
    step()
    o["Y"] = gemm.gemm(o["X"], d["W"], mode=F32_F16X2)                                 # fp32 C as F16X2 A
    step()
    o["Z"] = gemm.gemm(o["Y"].t(), d["W2"], mode=F32_TF32)                             # ... as transposed TF32 A
    step()
    o["S"] = gemm.gemm(o["Z"], d["W3"].t(), mode=F32_STRICT)                           # ... as STRICT A, B^T copied
    step()
    offs = torch.cumsum(d["counts"], 0, dtype=torch.int32)                             # written just before the call
    o["G"] = torch.full((m, 64), float("nan"), device="cuda")
    gemm.gemm(o["H"], d["Wg"], o["G"], offs=offs)
    step()
    a8, b8, b8b, scales, bias8 = d["s8"]
    o["Q"] = gemm.gemm_s8s8_requant(a8, b8, scales, bias8)
    step()
    o["R"] = gemm.gemm_s8s32(o["Q"], b8b)                                              # requant output as int8 A
    o["R_split"] = last_schedule(lib)[1]
    step()
    torch.cuda.synchronize()
    return o


@gpu
def test_dependent_chains(gemm, oracle, hooks, sms):
    """bf16 C as the next bf16 operand and as beta * C, a bias made by a torch kernel, fp32 C into F16X2 / transposed
    TF32 / STRICT with B^T, grouped offsets written by a torch kernel just before the call, int8 requant output as
    the next int8 operand: no synchronise in between, one after every call, and with PDL off give the same bits, and
    the dyadic steps their exact answers."""
    lib = hooks
    lib.b200_gemm_debug_set_bn(BN)
    d = chain_inputs(oracle)
    torch.cuda.synchronize()
    runs = [run_chain(gemm, d, False), run_chain(gemm, d, True)]
    lib.b200_gemm_debug_set_pdl(0)
    runs.append(run_chain(gemm, d, False))
    lib.b200_gemm_debug_set_pdl(1)
    base = runs[0]
    for r, o in enumerate(runs[1:], 1):
        for key in ("H", "E", "bias", "X", "Y", "Z", "S", "G", "Q", "R"):
            assert same_bits(o[key], base[key]), (r, key)
    assert base["X_split"] == 2 and base["R_split"] == 2
    dd = lambda t: t.double()
    H, E0, bias = base["H"], base["E0"], base["bias"]
    assert torch.equal(dd(H), (dd(d["A0"]) @ dd(d["B0"])))                             # |sums| <= 192: exact in bf16
    assert torch.equal(dd(E0), (dd(d["A0"]) @ dd(d["B0b"])))
    D = (dd(H) @ dd(d["B1"]) + 0.5 * dd(E0) + dd(bias)).clamp(min=0)
    assert torch.equal(D.float().double(), D)                                          # exact in fp32 before rounding
    assert same_bits(base["E"], D.float().bfloat16())
    X = dd(base["E"]) @ dd(d["B2"])
    assert torch.equal(X.float().double(), X) and same_bits(base["X"], X.float())
    ends = [int(e) for e in np.cumsum(GROUP_ROWS)]
    G = base["G"]
    for g, (lo, hi) in enumerate(zip([0] + ends[:-1], ends)):
        assert same_bits(G[lo:hi], (dd(H[lo:hi]) @ dd(d["Wg"][g])).float()), g
    assert ends[-1] < G.shape[0] and bool(torch.isnan(G[ends[-1]:]).all())
    # the fp32 modes on chained (not known-answer) operands: a sanity bound; the bits are pinned across the runs above
    for key, (A, B, tol) in {"Y": (base["X"], d["W"], 1e-4), "Z": (base["Y"].t(), d["W2"], 4e-3),
                             "S": (base["Z"], d["W3"].t(), 1e-4)}.items():
        t = dd(A) @ dd(B)
        assert float((dd(base[key]) - t).abs().max()) <= tol * float(t.abs().max()), key
    assert same_bits(base["Q"], d["s8_want"][0]) and same_bits(base["R"], d["s8_want"][1])


# ==== e. workspace across streams ===================================================================================
def f32_operands(m, n, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand((m, k), device="cuda", generator=g) * 2 - 1, torch.rand((k, n), device="cuda", generator=g) * 2 - 1


@gpu
def test_workspace_across_streams(gemm, hooks):
    """A transposing TF32 call on S1 interleaved with F16X2 calls on S2 that fork B's pre-pass onto the auxiliary
    stream; then the workspace regrown (b200_gemm_reserve_workspace, 4 GiB, more than any other test asks for; the
    process keeps it) while a long F16X2 call is still queued on S2.  Every result must be bit-identical to the same
    call run alone after a synchronise."""
    lib = hooks
    calls = []
    for i in range(4):
        A, B = f32_operands(520, 264, 328, 40 + i)
        calls.append(("tf32_tn", A.t().contiguous().t(), B, F32_TF32))
        A, B = f32_operands(1536, 1536, 1536, 50 + i)
        assert 1536 * 1536 * 2 >= 4e6                       # m k + k n: the pre-pass of B forks
        calls.append(("f16x2", A, B, F32_F16X2))
    big = f32_operands(4096, 4096, 4096, 60)
    after = [f32_operands(1536, 1536, 1536, 61), f32_operands(520, 264, 328, 62)]
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    forked(s1, s2)
    outs = []
    for name, A, B, mode in calls:
        with torch.cuda.stream(s1 if name == "tf32_tn" else s2):
            outs.append(gemm.gemm(A, B, mode=mode))
    with torch.cuda.stream(s2):
        big_out = gemm.gemm(*big, mode=F32_F16X2)
    assert lib.b200_gemm_reserve_workspace(4 << 30) == 0
    with torch.cuda.stream(s1):
        after_outs = [gemm.gemm(*after[0], mode=F32_F16X2), gemm.gemm(after[1][0].t().contiguous().t(), after[1][1],
                                                                       mode=F32_TF32)]
    joined(s1, s2)
    for (name, A, B, mode), got in zip(calls, outs):
        alone = gemm.gemm(A, B, mode=mode)
        torch.cuda.synchronize()
        assert same_bits(got, alone), name
    assert same_bits(big_out, gemm.gemm(*big, mode=F32_F16X2))
    assert same_bits(after_outs[0], gemm.gemm(*after[0], mode=F32_F16X2))
    assert same_bits(after_outs[1], gemm.gemm(after[1][0].t().contiguous().t(), after[1][1], mode=F32_TF32))


# ==== f. tensor-map cache ===========================================================================================
def exact16(A, B):
    return (A.double() @ B.double()).float()


@gpu
def test_tensor_map_cache(gemm, hooks):
    """More than 64 distinct tensor maps between two uses of one operand, and one address reused by operands of
    another shape, dtype or pitch (as when torch hands a freed block to the next tensor): every result stays exact."""
    X = dev(dyadic((256, 192), 20), torch.bfloat16)
    W = dev(dyadic((192, 136), 21), torch.bfloat16)
    first = gemm.gemm(X, W)
    others = [(dev(dyadic((64, 64 + 8 * (i % 4)), 100 + i), torch.bfloat16),
               dev(dyadic((64 + 8 * (i % 4), 72), 200 + i), torch.bfloat16)) for i in range(40)]
    for A, B in others:                                     # 80 maps
        assert same_bits(gemm.gemm(A, B), exact16(A, B))
    again = gemm.gemm(X, W)
    assert same_bits(first, exact16(X, W)) and same_bits(again, first)
    # one 16 KiB block read as a 64 x 128 bf16 A, then as 128 x 64, as fp16, and with 96 of 128 columns
    raw = torch.empty(64 * 128 * 2, dtype=torch.uint8, device="cuda")
    for i, (shape, dt, cols) in enumerate((((64, 128), torch.bfloat16, 128), ((128, 64), torch.bfloat16, 64),
                                           ((64, 128), torch.float16, 128), ((64, 128), torch.bfloat16, 96))):
        T = raw.view(dt).view(shape)
        assert T.data_ptr() == raw.data_ptr()
        T.copy_(dev(dyadic(shape, 30 + i), dt))
        V = T[:, :cols]
        Bv = dev(dyadic((cols, 64), 40 + i), dt)
        assert same_bits(gemm.gemm(V, Bv), exact16(V, Bv)), i
    # a freed operand's block handed to a tensor of another shape: when torch reuses the address, still exact
    T = torch.empty((64, 128), dtype=torch.bfloat16, device="cuda")
    T.copy_(dev(dyadic((64, 128), 50), torch.bfloat16))
    B = dev(dyadic((128, 64), 51), torch.bfloat16)
    assert same_bits(gemm.gemm(T, B), exact16(T, B))
    del T
    T = torch.empty((128, 64), dtype=torch.bfloat16, device="cuda")
    T.copy_(dev(dyadic((128, 64), 52), torch.bfloat16))
    B = dev(dyadic((64, 64), 53), torch.bfloat16)
    assert same_bits(gemm.gemm(T, B), exact16(T, B))


# ==== g. capture ====================================================================================================
@gpu
def test_captured_split_call_replays_bit_identical(gemm, hooks, sms):
    """A split-tail bf16 -> fp32 C call captured in a CUDA graph (no cross-stream wait or record under capture) and
    replayed twice gives the eager call's bits."""
    lib = hooks
    lib.b200_gemm_debug_set_bn(BN)
    job = job16(lib, "bf16", "nt", 3, sms, 900, 0.5)
    c0 = job.out.clone()
    torch.cuda.synchronize()
    assert job.run(lib, cur()) == (job.name, job.sched) and job.sched[1] == 3
    torch.cuda.synchronize()
    job.check("eager")
    eager = job.out.clone()
    job.out.copy_(c0)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    forked(s)
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            assert job.run(lib, cur()) == (job.name, job.sched)
    torch.cuda.synchronize()
    for r in range(2):
        job.out.copy_(c0)
        g.replay()
        torch.cuda.synchronize()
        assert same_bits(job.out, eager), r
    del g
