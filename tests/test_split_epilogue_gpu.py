"""The F16X2 kernel's deferred store (gemm_tc_split_kernel): a tile's C is stored while the tensor cores already run the
next tile's first k-blocks, unless the tile needs the general store or its CTA has no next tile.

Known-answer operands: small integers, which F16X2 scales by powers of two into fp16 without a low plane and sums
exactly, so C must equal the float64 product bit for bit whatever the schedule.  The shapes give every CTA several
tiles, mix whole tiles with edge tiles, put a K-split part after a whole tile, take C += A*B and beta != 0, and read
each operand layout; the chunk lengths put the first chunk of a tile below, at and above the k-blocks issued ahead of
a store.  Output buffers start as NaN so that a tile stored from the wrong sum, or not at all, cannot pass."""
import pytest

import _libs

try:
    import torch
except ImportError:
    torch = None

pytestmark = pytest.mark.gpu

OP_N, OP_T = 0, 1
CHUNKS = [-1, 32, 64, 96, 128, 160]          # elements of K per chunk (one k-block is 32), -1: the built-in 1024


@pytest.fixture(scope="module")
def g():
    return _libs.load_pkg()


@pytest.fixture
def chunk_hook(g):
    yield g.lib.b200_gemm_debug_set_split_chunk
    g.lib.b200_gemm_debug_set_split_chunk(-1, -1)


def ints(rows, cols, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-3, 4, (rows, cols), device="cuda", generator=gen).float()


def f16x2(g, A, B, C0=None, alpha=1.0, beta=0.0, op_a=OP_N, op_b=OP_N):
    """C = alpha * A B + beta * C0 through b200_gemm_f32_op in F16X2 mode, A and B given as op_a(A), op_b(B) stores."""
    m, k = A.shape
    n = B.shape[1]
    As = A.t().contiguous() if op_a else A.contiguous()
    Bs = B.t().contiguous() if op_b else B.contiguous()
    out = torch.full((m, n), float("nan"), device="cuda") if C0 is None else C0.clone()
    rc = g.lib.b200_gemm_f32_op(op_a, op_b, m, n, k, alpha, As.data_ptr(), As.stride(0), Bs.data_ptr(), Bs.stride(0),
                                beta, out.data_ptr(), out.stride(0), g.F32_F16X2, None)
    assert rc == 0, rc
    assert g.last_kernel().startswith("tc_f16x2"), g.last_kernel()
    return out


def exact(A, B, C0=None, alpha=1.0, beta=0.0):
    t = alpha * (A.double() @ B.double())
    if C0 is not None and beta != 0.0:
        t = t + beta * C0.double()
    return t.float()


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("shape", ["whole", "edges"])
def test_deferred_store_known_answer(g, chunk_hook, shape, chunk):
    """Several tiles per CTA: whole 128 x 128 tiles only, or with M / N edge tiles and a partial last k-block."""
    n_sm = sms()
    # whole: four rounds of tiles when the SM count is even; edges: a K-split last round as well
    m, n, k = (128 * 8, 128 * (n_sm // 2), 512) if shape == "whole" else (128 * 17 + 96, 128 * 17 + 40, 530)
    chunk_hook(chunk, chunk)
    A, B = ints(m, k, 11), ints(k, n, 12)
    assert torch.equal(f16x2(g, A, B), exact(A, B)), (shape, chunk)


@pytest.mark.parametrize("chunk", [-1, 64, 96])
def test_deferred_store_before_split_parts(g, chunk_hook, chunk):
    """One round of whole tiles, then a last round cut into K parts: each CTA's whole tile is stored behind the first
    k-blocks of its K part, and the parts fold into C in order."""
    n_sm = sms()
    m, n, k = 128 * (n_sm + n_sm // 4), 128, 1024
    chunk_hook(chunk, chunk)
    A, B = ints(m, k, 21), ints(k, n, 22)
    assert torch.equal(f16x2(g, A, B), exact(A, B)), chunk


@pytest.mark.parametrize("beta", [0.0, 0.5])
def test_deferred_store_general_epilogues(g, chunk_hook, beta):
    """alpha / beta and C += A*B take the general store for every tile."""
    m, n, k = 128 * 16, 128 * 20, 256
    A, B = ints(m, k, 31), ints(k, n, 32)
    C0 = ints(m, n, 33)
    assert torch.equal(f16x2(g, A, B, C0, alpha=2.0, beta=beta), exact(A, B, C0, 2.0, beta)), beta
    out = C0.clone()
    g.gemm_f32(A, B, out=out, mode=g.F32_F16X2, accumulate=True)
    assert g.last_kernel().startswith("tc_f16x2"), g.last_kernel()
    assert torch.equal(out, exact(A, B, C0, 1.0, 1.0))


@pytest.mark.parametrize("op_a,op_b", [(OP_N, OP_T), (OP_T, OP_N), (OP_T, OP_T)], ids=["NT", "TN", "TT"])
def test_deferred_store_layouts(g, chunk_hook, op_a, op_b):
    """The kernel's four layout instantiations (NN above) with several tiles per CTA and edge tiles."""
    m, n, k = 128 * 17 + 64, 128 * 18, 384
    A, B = ints(m, k, 41), ints(k, n, 42)
    assert torch.equal(f16x2(g, A, B, op_a=op_a, op_b=op_b), exact(A, B))
