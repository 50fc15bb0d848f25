"""how-to-optimize-gemm_b200 — Python host binding of libb200gemm.so (ctypes over the C ABI).

The product is the CUDA library; this module only loads it and forwards pointers.  PyTorch is
plumbing (device memory, streams, torch.distributed) and is imported lazily, only by the helpers
that take tensors.  There is NO CPU fallback: if the shared library is missing, import fails
loudly; if no sm_90 GPU is present, every compute call raises B200GemmError(-2).

Interface mirrored from the reference (file:line in /root/reference):
  MY_MMult(m, n, k, a, lda, b, ldb, c, ldc)                 aarch64/MMult0.cpp:3   (host, C += A*B)
  MY_MMult_cuda(handle, m, n, k, dA, lda, dB, ldb, dC, ldc)  cuda/test_MMult.cpp:13 (device, C = A*B)
  MY_MMult_int8(m, n, k, a, lda, b, ldb, c, ldc)             aarch64-int8/test_MMult.c:9
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200gemm.so")

F32_STRICT, F32_TF32, F32_BF16X3, F32_BF16X2, F32_AUTO, F32_F16X2 = 0, 1, 2, 3, 4, 5
OUT_F32, OUT_BF16, OUT_F16 = 0, 1, 2
OP_N, OP_T = 0, 1
ACT_NONE, ACT_RELU, ACT_GELU, ACT_GELU_TANH = 0, 1, 2, 3
ACTIVATIONS = {None: ACT_NONE, "relu": ACT_RELU, "gelu": ACT_GELU, "gelu_tanh": ACT_GELU_TANH}
FP8_E4M3, FP8_E5M2 = 0, 1

EXPORTS = [
    "b200_gemm_version", "b200_gemm_device_ok", "b200_gemm_strerror", "b200_gemm_last_kernel",
    "b200_gemm_launch_count", "b200_gemm_default_f32_mode", "b200_gemm_set_default_f32_mode",
    "b200_gemm_f32", "b200_gemm_f32_acc", "b200_gemm_f32_ex", "b200_gemm_workspace_bytes", "b200_gemm_reserve_workspace", "b200_mxf4_q_bytes", "b200_mxf4_sf_bytes",
    "b200_mxf4_quantize_a", "b200_mxf4_quantize_b", "b200_gemm_mxf4", "b200_gemm_f32_host", "b200_gemm_bf16", "b200_gemm_f16", "b200_gemm_s8s32",
    "b200_gemm_s8s32_host", "b200_gemm_s8s8_requant", "b200_gemm_f32_pack_b", "b200_gemm_f32_packed",
    "b200_gemm_f32_pack_free", "b200_gemm_f32_op", "b200_gemm_bf16_op", "b200_gemm_bf16_ex", "b200_gemm_f16_ex",
    "b200_gemm_bf16_epi", "b200_gemm_f16_epi", "b200_gemm_bf16_batched", "b200_gemm_f16_batched",
    "b200_gemm_bf16_grouped", "b200_gemm_f16_grouped", "b200_gemm_bf16_grouped_k", "b200_gemm_f16_grouped_k",
    "b200_gemm_s8s32_op", "b200_gemm_workspace_bytes_op", "b200_gemm_fp8", "b200_gemm_fp8_blockwise",
    "b200_gemm_fp8_grouped", "b200_gemm_fp8_batched", "b200_gemm_fp8_blockwise_grouped", "b200_gemm_fp8_blockwise_batched",
    "b200_gemm_fp8_q8", "b200_gemm_fp8_blockwise_q8", "b200_gemm_fp8_grouped_q8", "b200_gemm_fp8_batched_q8",
    "b200_gemm_fp8_blockwise_grouped_q8", "b200_gemm_fp8_blockwise_batched_q8", "b200_fp8_quantize",
    "b200_nccl_load", "b200_nccl_last_error", "b200_comm_unique_id", "b200_comm_init_rank",
    "b200_comm_destroy", "b200_rowpanel_create", "b200_rowpanel_destroy", "b200_rowpanel_slices", "b200_rowpanel_set_reserve_sms", "b200_rowpanel_trace", "b200_rowpanel_trace_dump", "b200_gemm_f32_rowpanel",
    "b200_gemm_f32_rowpanel_host", "b200_gemm_f32_pack_a", "b200_gemm_f32_packed_ab", "b200_gemm_f32_pack_free_a",
    "b200_convert_f32_to_bf16", "b200_gemm_debug_set_b_desc", "b200_gemm_debug_set_bn",
    "b200_gemm_debug_set_split_chunk", "b200_gemm_debug_kernel_timing", "b200_gemm_debug_kernel_time_ms",
    "b200_gemm_debug_set_cta_group", "b200_gemm_debug_set_split_tail", "b200_gemm_debug_last_schedule", "b200_gemm_debug_set_group_rows",
    "b200_gemm_debug_set_ffma_variant", "b200_gemm_debug_set_epilogue", "b200_gemm_debug_set_pdl", "b200_gemm_debug_set_dynamic_sched",
]


class B200GemmError(RuntimeError):
    def __init__(self, code, what=""):
        self.code = code
        super().__init__(f"b200gemm error {code}: {what}")


if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(nvcc, sm_90a). There is no CPU or PyTorch fallback for this path.")

lib = C.CDLL(LIB_PATH)
_vp, _i = C.c_void_p, C.c_int
lib.b200_gemm_version.restype = C.c_char_p
lib.b200_gemm_strerror.restype = C.c_char_p
lib.b200_gemm_strerror.argtypes = [_i]
lib.b200_gemm_last_kernel.restype = C.c_char_p
lib.b200_gemm_launch_count.restype = C.c_ulonglong
lib.b200_gemm_f32.argtypes = [_i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _vp]
lib.b200_gemm_f32_acc.argtypes = [_i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _vp]
lib.b200_gemm_f32_ex.argtypes = [_i, _i, _i, C.c_float, _vp, _i, _vp, _i, C.c_float, _vp, _i, _i, _vp]
lib.b200_gemm_workspace_bytes.argtypes = [_i, _i, _i, _i]
lib.b200_gemm_workspace_bytes.restype = C.c_size_t
lib.b200_gemm_reserve_workspace.argtypes = [C.c_size_t]
lib.b200_mxf4_q_bytes.argtypes = [_i, _i]
lib.b200_mxf4_q_bytes.restype = C.c_size_t
lib.b200_mxf4_sf_bytes.argtypes = [_i, _i]
lib.b200_mxf4_sf_bytes.restype = C.c_size_t
lib.b200_mxf4_quantize_a.argtypes = [_i, _i, _vp, _i, _vp, _vp, _vp]
lib.b200_mxf4_quantize_b.argtypes = [_i, _i, _vp, _i, _vp, _vp, _vp]
lib.b200_gemm_mxf4.argtypes = [_i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp]
lib.b200_gemm_f32_host.argtypes = [_i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i]
lib.b200_gemm_bf16.argtypes = [_i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _vp]
lib.b200_gemm_f16.argtypes = [_i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _vp]
lib.b200_gemm_s8s32.argtypes = [_i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _vp]
lib.b200_gemm_s8s32_host.argtypes = [_i, _i, _i, _vp, _i, _vp, _i, _vp, _i]
lib.b200_gemm_f32_op.argtypes = [_i, _i, _i, _i, _i, C.c_float, _vp, _i, _vp, _i, C.c_float, _vp, _i, _i, _vp]
lib.b200_gemm_bf16_op.argtypes = [_i, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _vp]
lib.b200_gemm_bf16_ex.argtypes = [_i, _i, _i, _i, _i, C.c_float, _vp, _i, _vp, _i, C.c_float, _vp, _i, _i, _vp]
lib.b200_gemm_f16_ex.argtypes = [_i, _i, _i, _i, _i, C.c_float, _vp, _i, _vp, _i, C.c_float, _vp, _i, _i, _vp]
lib.b200_gemm_bf16_epi.argtypes = [_i, _i, _i, _i, _i, C.c_float, _vp, _i, _vp, _i, C.c_float, _vp, _i, _i, _vp, _i, _vp]
lib.b200_gemm_f16_epi.argtypes = [_i, _i, _i, _i, _i, C.c_float, _vp, _i, _vp, _i, C.c_float, _vp, _i, _i, _vp, _i, _vp]
_ll = C.c_longlong
lib.b200_gemm_bf16_batched.argtypes = [_i, _i, _i, _i, _i, C.c_float, _vp, _i, _ll, _vp, _i, _ll, C.c_float, _vp, _i, _ll,
                                       _i, _i, _vp]
lib.b200_gemm_f16_batched.argtypes = [_i, _i, _i, _i, _i, C.c_float, _vp, _i, _ll, _vp, _i, _ll, C.c_float, _vp, _i, _ll,
                                      _i, _i, _vp]
lib.b200_gemm_bf16_grouped.argtypes = [_i, _i, _i, _i, C.c_float, _vp, _i, _vp, _i, _ll, _vp, _i, C.c_float, _vp, _i, _i,
                                       _vp]
lib.b200_gemm_f16_grouped.argtypes = [_i, _i, _i, _i, C.c_float, _vp, _i, _vp, _i, _ll, _vp, _i, C.c_float, _vp, _i, _i,
                                      _vp]
lib.b200_gemm_bf16_grouped_k.argtypes = [_i, _i, _i, _i, _i, C.c_float, _vp, _i, _vp, _i, _vp, _i, C.c_float, _vp, _i, _ll,
                                         _i, _vp]
lib.b200_gemm_f16_grouped_k.argtypes = [_i, _i, _i, _i, _i, C.c_float, _vp, _i, _vp, _i, _vp, _i, C.c_float, _vp, _i, _ll,
                                        _i, _vp]
lib.b200_gemm_s8s32_op.argtypes = [_i, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _vp]
lib.b200_gemm_workspace_bytes_op.argtypes = [_i, _i, _i, _i, _i, _i]
lib.b200_gemm_fp8.argtypes = [_i, _i, _i, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _vp]
lib.b200_gemm_fp8_blockwise.argtypes = [_i, _i, _i, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _ll, _ll, _vp, _i, _ll, _ll,
                                        _vp, _vp, _i, _i, _vp]
lib.b200_gemm_fp8_grouped.argtypes = [_i, _i, _i, _i, _i, _vp, _i, _vp, _i, _ll, _vp, _i, _vp, _vp, _ll, _vp, _i, _i, _i,
                                      _vp]
lib.b200_gemm_fp8_batched.argtypes = [_i, _i, _i, _i, _i, _vp, _i, _ll, _vp, _i, _ll, _vp, _ll, _vp, _ll, _vp, _i, _ll,
                                      _i, _i, _i, _vp]
lib.b200_gemm_fp8_blockwise_grouped.argtypes = [_i, _i, _i, _i, _i, _vp, _i, _vp, _i, _ll, _vp, _i, _vp, _ll, _ll, _vp, _i,
                                                _ll, _ll, _ll, _vp, _i, _i, _vp]
lib.b200_gemm_fp8_blockwise_batched.argtypes = [_i, _i, _i, _i, _i, _vp, _i, _ll, _vp, _i, _ll, _vp, _i, _ll, _ll, _ll, _vp,
                                                _i, _ll, _ll, _ll, _vp, _i, _ll, _i, _i, _vp]
lib.b200_gemm_fp8_q8.argtypes = [_i, _i, _i, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _vp, _i, _vp,
                                 _vp, _ll, _ll, _vp]
lib.b200_gemm_fp8_blockwise_q8.argtypes = [_i, _i, _i, _i, _i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _ll, _ll, _vp, _i, _ll,
                                           _ll, _vp, _i, _i, _vp, _i, _vp, _vp, _ll, _ll, _vp]
lib.b200_gemm_fp8_grouped_q8.argtypes = [_i, _i, _i, _i, _i, _vp, _i, _vp, _i, _ll, _vp, _i, _vp, _vp, _ll, _i, _i, _i, _vp,
                                         _i, _vp, _ll, _ll, _vp]
lib.b200_gemm_fp8_batched_q8.argtypes = [_i, _i, _i, _i, _i, _vp, _i, _ll, _vp, _i, _ll, _vp, _ll, _vp, _ll, _i, _i, _i,
                                         _vp, _i, _ll, _vp, _ll, _ll, _ll, _i, _vp]
lib.b200_gemm_fp8_blockwise_grouped_q8.argtypes = [_i, _i, _i, _i, _i, _vp, _i, _vp, _i, _ll, _vp, _i, _vp, _ll, _ll, _vp,
                                                   _i, _ll, _ll, _ll, _i, _i, _vp, _i, _vp, _ll, _ll, _vp]
lib.b200_gemm_fp8_blockwise_batched_q8.argtypes = [_i, _i, _i, _i, _i, _vp, _i, _ll, _vp, _i, _ll, _vp, _i, _ll, _ll, _ll,
                                                   _vp, _i, _ll, _ll, _ll, _i, _i, _vp, _i, _ll, _vp, _ll, _ll, _ll, _i,
                                                   _vp]
lib.b200_fp8_quantize.argtypes = [_i, _i, _i, _i, _i, _i, _vp, _i, _ll, _vp, _i, _ll, _vp, _ll, _ll, _ll, _vp, _i, _ll, _vp,
                                  _ll, _ll, _ll, _vp]
lib.b200_gemm_workspace_bytes_op.restype = C.c_size_t
lib.b200_gemm_f32_pack_b.argtypes = [_i, _i, _vp, _i, _i, C.POINTER(_vp), _vp]
lib.b200_gemm_f32_packed.argtypes = [_i, _i, _i, _vp, _i, _vp, _vp, _i, _i, _vp]
lib.b200_gemm_f32_pack_free.argtypes = [_vp]
lib.b200_gemm_f32_pack_free.restype = None
lib.b200_gemm_f32_pack_a.argtypes = [_i, _i, _vp, _i, _i, C.POINTER(_vp), _vp]
lib.b200_gemm_f32_packed_ab.argtypes = [_i, _i, _i, _vp, _i, _vp, _vp, _i, _i, _vp]
lib.b200_gemm_f32_pack_free_a.argtypes = [_vp]
lib.b200_gemm_f32_pack_free_a.restype = None
lib.b200_nccl_load.argtypes = [C.c_char_p]
lib.b200_nccl_last_error.restype = C.c_char_p
lib.b200_comm_unique_id.argtypes = [_vp]
lib.b200_comm_init_rank.argtypes = [C.POINTER(_vp), _vp, _i, _i]
lib.b200_comm_destroy.argtypes = [_vp]
lib.b200_rowpanel_create.argtypes = [C.POINTER(_vp), _vp, _i, _i, _i, _i, C.POINTER(_i), _i]
lib.b200_rowpanel_destroy.argtypes = [_vp]
lib.b200_rowpanel_destroy.restype = None
lib.b200_rowpanel_slices.argtypes = [_vp, C.POINTER(_i), _i]
lib.b200_rowpanel_set_reserve_sms.argtypes = [_vp, _i]
lib.b200_rowpanel_trace.argtypes = [_vp, _i]
lib.b200_rowpanel_trace.restype = None
lib.b200_rowpanel_trace_dump.argtypes = [_vp, C.POINTER(C.c_float), _i]
lib.b200_gemm_f32_rowpanel.argtypes = [_vp, _i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _vp]
lib.b200_gemm_f32_rowpanel_host.argtypes = [_vp, _i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i]
lib.b200_gemm_s8s8_requant.argtypes = [_i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _vp]
lib.b200_convert_f32_to_bf16.argtypes = [_vp, _vp, C.c_size_t, _vp]
lib.b200_gemm_debug_set_b_desc.argtypes = [_i, _i]
lib.b200_gemm_set_default_f32_mode.argtypes = [_i]
lib.b200_gemm_debug_set_bn.argtypes = [_i]
lib.b200_gemm_debug_set_split_chunk.argtypes = [_i, _i]
lib.b200_gemm_debug_kernel_timing.argtypes = [_i]
lib.b200_gemm_debug_set_cta_group.argtypes = [_i]
lib.b200_gemm_debug_set_split_tail.argtypes = [_i]
lib.b200_gemm_debug_last_schedule.argtypes = [C.POINTER(_i)] * 4
lib.b200_gemm_debug_last_schedule.restype = None
lib.b200_gemm_debug_set_pdl.argtypes = [_i]
lib.b200_gemm_debug_set_dynamic_sched.argtypes = [_i]
lib.b200_gemm_debug_kernel_time_ms.argtypes = [C.POINTER(C.c_double)]


def kernel_time_ms():
    """(sum_ms, launches) of the dominant GEMM kernel since kernel timing was enabled."""
    s = C.c_double(0.0)
    n = lib.b200_gemm_debug_kernel_time_ms(C.byref(s))
    return s.value, n


def _check(rc):
    if rc != 0:
        what = lib.b200_gemm_strerror(rc).decode()
        if rc == -5:
            what += ": " + lib.b200_nccl_last_error().decode()
        raise B200GemmError(rc, what)


def version():
    return lib.b200_gemm_version().decode()


def last_kernel():
    return lib.b200_gemm_last_kernel().decode()


def launch_count():
    return int(lib.b200_gemm_launch_count())


def _stream_ptr(stream):
    if stream is None:
        import torch
        return torch.cuda.current_stream().cuda_stream
    return getattr(stream, "cuda_stream", stream)


# ---- raw-pointer forms (exact mirrors of the reference signatures) ------------------------------
def MY_MMult_cuda(handle, m, n, k, dA, lda, dB, ldb, dC, ldc, mode=F32_AUTO, stream=0):
    """cuda/test_MMult.cpp:13-14 — device pointers (ints), C = A*B.  `handle` is ignored, as the
    reference's hand kernels ignore it (cuda/MMult_cuda_12.cu:228)."""
    _check(lib.b200_gemm_f32(m, n, k, dA, lda, dB, ldb, dC, ldc, mode, stream))


def MY_MMult(m, n, k, a, lda, b, ldb, c, ldc, mode=F32_AUTO):
    """aarch64/MMult0.cpp:3-4 — numpy float32 host arrays, C += A*B in place."""
    _check(lib.b200_gemm_f32_host(m, n, k, a.ctypes.data, lda, b.ctypes.data, ldb, c.ctypes.data, ldc, mode))


def MY_MMult_int8(m, n, k, a, lda, b, ldb, c, ldc):
    """aarch64-int8/test_MMult.c:9,98 — numpy int8 host arrays, int32 C = A*B."""
    _check(lib.b200_gemm_s8s32_host(m, n, k, a.ctypes.data, lda, b.ctypes.data, ldb, c.ctypes.data, ldc))


# ---- tensor forms (torch CUDA tensors; row-major, last dim contiguous) --------------------------
def _ld(t):
    assert t.dim() == 2 and (t.stride(1) == 1 or t.shape[1] <= 1), "row-major 2-D tensor with unit inner stride expected"
    if t.shape[1] <= 1:              # a single column: any stride is reported for the size-1 dimension
        return max(1, t.stride(0)) if t.shape[0] > 1 else 1
    return t.stride(0) if t.shape[0] > 1 else max(t.shape[1], t.stride(0))


def operand_layout(shape, strides):
    """(op, ld) under which the C ABI reads a 2-D operand of this shape and these strides (elements) in place.

    Row-major (unit stride along dim 1): OP_N, ld = stride(0).  Transposed view of a row-major matrix (unit stride
    along dim 0, e.g. W.t()): OP_T, ld = stride(1).  A dimension of size 1 may have any stride; a tensor that is both
    (a single row or column) is taken as row-major.  Any other stride pattern raises ValueError: the library never
    copies an operand."""
    r, c = shape
    s0, s1 = strides
    if c <= 1:                       # a single column: row-major with any row stride
        return OP_N, (max(1, s0) if r > 1 else 1)
    if s1 == 1:
        return OP_N, (s0 if r > 1 else max(c, s0))
    if s0 == 1 or r <= 1:            # column c of the view is row c of the stored (c x r) matrix
        return OP_T, s1
    raise ValueError(f"operand of shape {tuple(shape)} and strides {tuple(strides)} is neither row-major nor the "
                     "transpose of a row-major matrix")


def batched_operand_layout(shape, strides):
    """(op, ld, batch stride) under which the C ABI's batched entry points read a 3-D operand (batch, rows, cols) in
    place: the last two dimensions resolve as operand_layout does, the batch stride is stride(0) (0 for an expand()ed
    operand, which is broadcast over the batch; 0 as well for a batch of one, whose stride is never used)."""
    op, ld = operand_layout(tuple(shape[1:]), tuple(strides[1:]))
    return op, ld, (strides[0] if shape[0] > 1 else 0)


def _gemm_batched(A, B, out, alpha, beta, bias, activation, out_dtype, stream):
    """gemm() on 3-D operands: C[b] = alpha * A[b] @ B[b] + beta * C[b] in one call (b200_gemm_*_batched)."""
    import torch
    if A.dtype != B.dtype:
        raise TypeError(f"operands of different dtypes: {A.dtype} and {B.dtype}")
    if A.dtype not in (torch.bfloat16, torch.float16):
        raise TypeError(f"batched (3-D) operands must be bf16 or fp16, not {A.dtype}")
    if bias is not None or activation is not None:
        raise ValueError("the batched GEMM has no bias / activation epilogue")
    if A.dim() != 3 or B.dim() != 3:
        raise ValueError(f"batched operands must both be 3-D (pass an expand()ed view to broadcast one), not "
                         f"{A.dim()}-D and {B.dim()}-D")
    batch, m, k = A.shape
    batch_b, k2, n = B.shape
    if batch_b != batch:
        raise ValueError(f"batch sizes differ: {batch} and {batch_b}")
    assert k == k2, (A.shape, B.shape)
    op_a, lda, sa = batched_operand_layout(tuple(A.shape), A.stride())
    op_b, ldb, sb = batched_operand_layout(tuple(B.shape), B.stride())
    cdt = out_dtype or (out.dtype if out is not None else torch.float32)
    assert cdt in (torch.float32, A.dtype), f"{A.dtype} operands write float32 or {A.dtype} C, not {cdt}"
    if out is None:
        assert beta == 0.0, "beta != 0 reads C: pass out"
        out = torch.empty((batch, m, n), dtype=cdt, device=A.device)
    assert out.dtype == cdt
    if out.dim() != 3 or tuple(out.shape) != (batch, m, n):
        raise ValueError(f"out must have shape {(batch, m, n)}, not {tuple(out.shape)}")
    if batch == 0:
        return out
    if (n > 1 and out.stride(2) != 1) or (m > 1 and out.stride(1) < n):
        raise ValueError("out must be row-major in its last two dimensions")
    ldc = _ld(out[0])
    sc = out.stride(0) if batch > 1 else 0
    assert A.is_cuda and B.is_cuda and out.is_cuda
    fn, ot = (lib.b200_gemm_bf16_batched, OUT_BF16) if A.dtype == torch.bfloat16 else (lib.b200_gemm_f16_batched, OUT_F16)
    _check(fn(op_a, op_b, m, n, k, alpha, A.data_ptr(), lda, sa, B.data_ptr(), ldb, sb, beta, out.data_ptr(), ldc, sc,
              batch, OUT_F32 if cdt == torch.float32 else ot, _stream_ptr(stream)))
    return out


def _check_offs(offs):
    import torch
    if not isinstance(offs, torch.Tensor) or offs.dtype != torch.int32 or offs.dim() != 1:
        raise ValueError("offs must be a 1-D int32 tensor")
    if not offs.is_contiguous():
        raise ValueError("offs must be contiguous")


def grouped_layout(A, B, offs):
    """(total_m, n, k, op_b, ldb, stride_b, groups) under which b200_gemm_*_grouped reads gemm(A, B, offs=offs) in place:
    A (total_m x k) row-major, B (groups x k x n) whose last two dimensions resolve as batched_operand_layout does (so
    W.transpose(-2, -1) of a (groups, n, k) weight is op_b = OP_T), offs a contiguous 1-D int32 tensor of groups
    cumulative end rows.  Raises ValueError for anything else, a broadcast or overlapping B included; the device of the
    tensors is not checked here."""
    if A.dim() != 2 or B.dim() != 3:
        raise ValueError(f"a grouped GEMM takes a 2-D A and a 3-D B, not {A.dim()}-D and {B.dim()}-D")
    _check_offs(offs)
    groups, k2, n = B.shape
    total_m, k = A.shape
    if offs.numel() != groups:
        raise ValueError(f"offs has {offs.numel()} elements for {groups} groups of B")
    if k2 != k:
        raise ValueError(f"inner dimensions differ: A is {tuple(A.shape)}, B is {tuple(B.shape)}")
    op_a, _ = operand_layout(tuple(A.shape), A.stride())
    if op_a != OP_N:
        raise ValueError("A of a grouped GEMM must be row-major")
    op_b, ldb, sb = batched_operand_layout(tuple(B.shape), B.stride())
    if groups > 1 and sb < (n if op_b == OP_T else k) * ldb:
        raise ValueError(f"the groups of B must not overlap or be broadcast (stride(0) = {B.stride(0)})")
    return total_m, n, k, op_b, ldb, sb, groups


def _gemm_grouped(A, B, out, offs, alpha, beta, bias, activation, out_dtype, stream):
    """gemm(A, B, offs=offs): rows [offs[g-1], offs[g]) of out = alpha * A[rows] @ B[g] + beta * out[rows], one launch
    (b200_gemm_*_grouped)."""
    import torch
    if A.dtype != B.dtype:
        raise TypeError(f"operands of different dtypes: {A.dtype} and {B.dtype}")
    if A.dtype not in (torch.bfloat16, torch.float16):
        raise TypeError(f"grouped operands must be bf16 or fp16, not {A.dtype}")
    if bias is not None or activation is not None:
        raise ValueError("the grouped GEMM has no bias / activation epilogue")
    total_m, n, k, op_b, ldb, sb, groups = grouped_layout(A, B, offs)
    cdt = out_dtype or (out.dtype if out is not None else torch.float32)
    if cdt not in (torch.float32, A.dtype):
        raise ValueError(f"{A.dtype} operands write float32 or {A.dtype} C, not {cdt}")
    if out is not None:
        if out.dtype != cdt:
            raise ValueError(f"out is {out.dtype}, not {cdt}")
        if out.dim() != 2 or tuple(out.shape) != (total_m, n):
            raise ValueError(f"out must have shape {(total_m, n)}, not {tuple(out.shape)}")
        if (n > 1 and out.stride(1) != 1) or (total_m > 1 and out.stride(0) < n):
            raise ValueError("out must be row-major")
    if not (A.is_cuda and B.is_cuda and offs.is_cuda and (out is None or out.is_cuda)):
        raise ValueError("A, B, offs and out must be CUDA tensors")
    if out is None:
        assert beta == 0.0, "beta != 0 reads C: pass out"
        out = torch.empty((total_m, n), dtype=cdt, device=A.device)
    fn, ot = (lib.b200_gemm_bf16_grouped, OUT_BF16) if A.dtype == torch.bfloat16 else (lib.b200_gemm_f16_grouped, OUT_F16)
    _check(fn(op_b, total_m, n, k, alpha, A.data_ptr(), _ld(A), B.data_ptr(), ldb, sb, offs.data_ptr(), groups, beta,
              out.data_ptr(), _ld(out), OUT_F32 if cdt == torch.float32 else ot, _stream_ptr(stream)))
    return out


def grouped_k_layout(A, B, offs):
    """(m, n, total_k, op_a, lda, op_b, ldb, groups) under which b200_gemm_*_grouped_k reads gemm(A, B, offs=offs) for a
    2-D A (m x total_k) and a 2-D B (total_k x n) in place: each resolves as operand_layout does (so dy.t() of a
    row-major dy is op_a = OP_T and a row-major x is op_b = OP_N), offs a contiguous 1-D int32 tensor of groups
    cumulative ends along K.  Raises ValueError for anything else; the device of the tensors is not checked here."""
    _check_offs(offs)
    m, total_k = A.shape
    k2, n = B.shape
    if k2 != total_k:
        raise ValueError(f"inner dimensions differ: A is {tuple(A.shape)}, B is {tuple(B.shape)}")
    op_a, lda = operand_layout(tuple(A.shape), A.stride())
    op_b, ldb = operand_layout(tuple(B.shape), B.stride())
    return m, n, total_k, op_a, lda, op_b, ldb, offs.numel()


def _gemm_grouped_k(A, B, out, offs, alpha, beta, bias, activation, out_dtype, stream):
    """gemm(A, B, offs=offs) with a 2-D B: out[g] = alpha * A[:, K_g] @ B[K_g, :] + beta * out[g] for the K ranges
    K_g = [offs[g-1], offs[g]), one launch (b200_gemm_*_grouped_k)."""
    import torch
    if A.dtype != B.dtype:
        raise TypeError(f"operands of different dtypes: {A.dtype} and {B.dtype}")
    if A.dtype not in (torch.bfloat16, torch.float16):
        raise TypeError(f"grouped operands must be bf16 or fp16, not {A.dtype}")
    if bias is not None or activation is not None:
        raise ValueError("the grouped GEMM has no bias / activation epilogue")
    m, n, total_k, op_a, lda, op_b, ldb, groups = grouped_k_layout(A, B, offs)
    cdt = out_dtype or (out.dtype if out is not None else torch.float32)
    if cdt not in (torch.float32, A.dtype):
        raise ValueError(f"{A.dtype} operands write float32 or {A.dtype} C, not {cdt}")
    if out is not None:
        if out.dtype != cdt:
            raise ValueError(f"out is {out.dtype}, not {cdt}")
        if out.dim() != 3 or tuple(out.shape) != (groups, m, n):
            raise ValueError(f"out must have shape {(groups, m, n)}, not {tuple(out.shape)}")
        if (n > 1 and out.stride(2) != 1) or (m > 1 and out.stride(1) < n):
            raise ValueError("out must be row-major in its last two dimensions")
        if groups > 1 and m * n > 0 and out.stride(0) < (m - 1) * out.stride(1) + n:
            raise ValueError(f"the groups of out must not overlap (stride(0) = {out.stride(0)})")
    if not (A.is_cuda and B.is_cuda and offs.is_cuda and (out is None or out.is_cuda)):
        raise ValueError("A, B, offs and out must be CUDA tensors")
    if out is None:
        assert beta == 0.0, "beta != 0 reads C: pass out"
        out = torch.empty((groups, m, n), dtype=cdt, device=A.device)
    if groups == 0:
        return out
    fn, ot = (lib.b200_gemm_bf16_grouped_k, OUT_BF16) if A.dtype == torch.bfloat16 else (lib.b200_gemm_f16_grouped_k, OUT_F16)
    _check(fn(op_a, op_b, m, n, total_k, alpha, A.data_ptr(), lda, B.data_ptr(), ldb, offs.data_ptr(), groups, beta,
              out.data_ptr(), _ld(out[0]), out.stride(0), OUT_F32 if cdt == torch.float32 else ot, _stream_ptr(stream)))
    return out


def _epilogue_args(A, B, bias, activation):
    """Checks a bias / activation request of gemm() (before anything touches the device); returns the ACT_* code."""
    import torch
    if activation not in ACTIVATIONS:
        raise ValueError(f"activation must be one of {sorted(a for a in ACTIVATIONS if a)} or None, not {activation!r}")
    if A.dtype not in (torch.bfloat16, torch.float16) or B.dtype != A.dtype:
        raise TypeError(f"a bias or an activation needs bf16 or fp16 operands of one dtype, not {A.dtype} and {B.dtype}")
    if bias is not None:
        if bias.dtype != A.dtype:
            raise ValueError(f"the bias must have the operands' dtype {A.dtype}, not {bias.dtype}")
        if bias.dim() != 1 or bias.shape[0] != B.shape[1]:
            raise ValueError(f"the bias must be 1-D with n = {B.shape[1]} elements, not of shape {tuple(bias.shape)}")
        if not bias.is_contiguous() or not bias.is_cuda:
            raise ValueError("the bias must be a contiguous CUDA tensor")
    return ACTIVATIONS[activation]


def gemm(A, B, out=None, *, offs=None, alpha=1.0, beta=0.0, bias=None, activation=None, mode=F32_AUTO,
         out_dtype=None, stream=None):
    """C = alpha * A @ B + beta * C for fp32 (any precision mode), bf16 (fp32 or bf16 C), fp16 (fp32 or fp16 C) and
    int8 (int32 C) CUDA tensors.  Each operand may be row-major or the transpose of a row-major matrix (x @ W.t()
    passes W as stored): it is read in place (b200_gemm_f32_op / _bf16_epi / _f16_epi / _s8s32_op), never
    copied.  out must be row-major; it is read only when beta != 0.  int8 takes alpha = 1, beta = 0 only.

    bf16 and fp16 also take a bias (1-D, contiguous, n elements of the operands' dtype) and an activation (None,
    "relu", "gelu" or "gelu_tanh") fused into the epilogue (b200_gemm_bf16_epi / _f16_epi):
    C = act(alpha * A @ B + beta * C + bias), so gemm(x, W.t(), bias=b, activation="gelu") is
    F.gelu(F.linear(x, W, b)) in one launch.  Other operand dtypes refuse them with TypeError; a bias of another dtype
    or length is a ValueError.

    3-D bf16 or fp16 operands (batch, rows, cols) with equal batch sizes are a strided batch, torch.bmm / baddbmm:
    out[b] = alpha * A[b] @ B[b] + beta * out[b] in one launch (b200_gemm_bf16_batched / _f16_batched).  The last two
    dimensions of each operand resolve as for 2-D operands and its batch stride is stride(0), so k.transpose(1, 2) and
    expand()ed operands (stride 0, broadcast) are read in place.  out is 3-D and row-major in its last two dimensions.
    3-D fp32 or int8 operands are a TypeError; a bias, an activation, unequal batch sizes or another out is a
    ValueError.

    offs (a contiguous 1-D int32 CUDA tensor, one cumulative end row per group) makes it a grouped GEMM,
    torch._grouped_mm(A, B, offs=offs): A is 2-D row-major (total_m x k), B is 3-D bf16 or fp16 (groups x k x n,
    W.transpose(-2, -1) of a (groups, n, k) weight read in place), and rows [offs[g-1], offs[g]) of out are
    alpha * A[rows] @ B[g] + beta * out[rows], every group in one launch (b200_gemm_bf16_grouped / _f16_grouped).  The
    offsets stay on the device (the call never synchronises).  out is row-major (total_m x n); a new one is
    torch.empty, so its rows from offs[-1] on are unspecified, as in torch.  out_dtype defaults to float32 as for every
    16-bit gemm() (torch._grouped_mm's default is the operands' dtype).  fp32 or int8 operands are a TypeError; a bias,
    an activation, another offs, A or out, or a broadcast or overlapping B is a ValueError.

    offs with a 2-D A and a 2-D B is torch._grouped_mm's 2-D x 2-D form, where the offsets split K: the weight gradient
    dW_g = dy_g^T x_g of such a layer is gemm(dy.t(), x, offs=offs).  A is m x total_k and B is total_k x n, each
    row-major or transposed and read in place; out[g] = alpha * A[:, K_g] @ B[K_g, :] + beta * out[g] for the K range
    K_g = [offs[g-1], offs[g]) (clamped as above, to total_k), every group in one launch (b200_gemm_bf16_grouped_k /
    _f16_grouped_k).  out is (groups, m, n), row-major in its last two dimensions, with out.stride(0) between groups;
    every group is written, an empty one with zeros (beta * out[g] when beta != 0).  out_dtype defaults to float32.
    The refusals are those of the grouped form, and an overlapping out is a ValueError."""
    import torch
    if offs is not None:
        if A.dim() == 2 and B.dim() == 2:
            return _gemm_grouped_k(A, B, out, offs, alpha, beta, bias, activation, out_dtype, stream)
        return _gemm_grouped(A, B, out, offs, alpha, beta, bias, activation, out_dtype, stream)
    if A.dim() == 3 or B.dim() == 3:
        return _gemm_batched(A, B, out, alpha, beta, bias, activation, out_dtype, stream)
    epi = bias is not None or activation is not None
    act = _epilogue_args(A, B, bias, activation) if epi else ACT_NONE
    assert A.dim() == 2 and B.dim() == 2 and A.is_cuda and B.is_cuda
    if A.dtype != B.dtype:
        raise TypeError(f"operands of different dtypes: {A.dtype} and {B.dtype}")
    m, k = A.shape
    k2, n = B.shape
    assert k == k2, (A.shape, B.shape)
    op_a, lda = operand_layout(tuple(A.shape), A.stride())
    op_b, ldb = operand_layout(tuple(B.shape), B.stride())
    if A.dtype == torch.float32:
        cdt = torch.float32
    elif A.dtype in (torch.bfloat16, torch.float16):
        cdt = out_dtype or (out.dtype if out is not None else torch.float32)
        assert cdt in (torch.float32, A.dtype), f"{A.dtype} operands write float32 or {A.dtype} C, not {cdt}"
    elif A.dtype == torch.int8:
        cdt = torch.int32
    else:
        raise TypeError(f"unsupported operand dtype {A.dtype}")
    if A.dtype == torch.int8 and (alpha != 1.0 or beta != 0.0):
        raise ValueError("the int8 GEMM takes alpha = 1, beta = 0 only")
    if out is None:
        assert beta == 0.0, "beta != 0 reads C: pass out"
        out = torch.empty((m, n), dtype=cdt, device=A.device)
    assert out.dtype == cdt and tuple(out.shape) == (m, n)
    if n > 1:
        assert out.stride(1) == 1, "out must be row-major"
    st = _stream_ptr(stream)
    if A.dtype == torch.float32:
        _check(lib.b200_gemm_f32_op(op_a, op_b, m, n, k, alpha, A.data_ptr(), lda, B.data_ptr(), ldb, beta, out.data_ptr(),
                                    _ld(out), mode, st))
    elif A.dtype in (torch.bfloat16, torch.float16):
        fn, ot = (lib.b200_gemm_bf16_epi, OUT_BF16) if A.dtype == torch.bfloat16 else (lib.b200_gemm_f16_epi, OUT_F16)
        _check(fn(op_a, op_b, m, n, k, alpha, A.data_ptr(), lda, B.data_ptr(), ldb, beta, out.data_ptr(), _ld(out),
                  OUT_F32 if cdt == torch.float32 else ot, bias.data_ptr() if bias is not None else None, act, st))
    else:
        _check(lib.b200_gemm_s8s32_op(op_a, op_b, m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb, out.data_ptr(), _ld(out), st))
    return out


def _fp8_type(t):
    import torch
    return {torch.float8_e4m3fn: FP8_E4M3, torch.float8_e5m2: FP8_E5M2}.get(t.dtype)


def _is_fp8(dtype):
    import torch
    return dtype in (torch.float8_e4m3fn, torch.float8_e5m2)


def _blockwise_recipe(scale_a, scale_b, m, n, k):
    """(scale_a_block, scale_b_block) of torch._scaled_mm's blockwise recipes, resolved from the scales' shapes in the
    order torch checks them, or None.  Both scales must be 2-D float32 tensors."""
    import torch
    if scale_a.dtype != torch.float32 or scale_b.dtype != torch.float32 or scale_a.dim() != 2 or scale_b.dim() != 2:
        return None
    q, mb, nb = -(-k // 128), -(-m // 128), -(-n // 128)
    sa, sb = tuple(scale_a.shape), tuple(scale_b.shape)
    for blocks, want_a, want_b in (((1, 128), (m, q), (q, nb)), ((1, 1), (m, q), (q, n)), ((128, 1), (mb, q), (q, n))):
        if sa == want_a and sb == want_b:
            return blocks
    return None


def scaled_mm(A, B, scale_a, scale_b, bias=None, out_dtype=None, use_fast_accum=False, out=None, stream=None, *,
              scale_result=None):
    """torch._scaled_mm for FP8 CUDA tensors: out = ((A @ B) * scale_a) * scale_b + bias, each step rounded in fp32 and
    the result rounded once to out_dtype (b200_gemm_fp8), or with blockwise scales the sum over 128-element k-blocks
    of each block's product times its scales (b200_gemm_fp8_blockwise).

    A (m x k) and B (k x n) are float8_e4m3fn or float8_e5m2 (not both e5m2), each row-major or the transpose of a
    row-major matrix and read in place; torch's layout is a row-major A and a column-major B (x @ W.t()).  scale_a and
    scale_b are float32 CUDA tensors: one element each (tensorwise), or scale_a (m, 1) and scale_b (1, n) (rowwise).
    Or, with q = ceil(k / 128), blockwise, as 2-D tensors of any non-negative strides:
      scale_a (m, q) with scale_b (q, ceil(n / 128))    1 x 128 activations, 128 x 128 weights (x @ W.t(), DeepSeek-V3)
      scale_a (m, q) with scale_b (q, n)                1 x 128 both (the weight gradient, K = tokens)
      scale_a (ceil(m / 128), q) with scale_b (q, n)    128 x 128 A, 1 x 128 B
    Each k-block's product is then added to an fp32 running sum with one fused multiply-add by rn(sa * sb); see
    b200_gemm_fp8_blockwise.  Where k <= 128 a blockwise shape can also be a tensorwise / rowwise one ((m, 1) with (1, 1)
    or (1, n)); such scales keep their tensorwise / rowwise meaning, whose rounding rn(rn(acc * sa) * sb) differs from
    the blockwise rn(acc * rn(sa * sb)).  The scales stay on the device: the call never synchronises.  bias: None or n
    contiguous elements of out_dtype.  out_dtype is torch.bfloat16 (the default), torch.float16 or torch.float32.
    use_fast_accum = False promotes the tensor core's FP8 sums to fp32 every 128 elements of K; True keeps one
    tensor-core accumulator over K (faster, less precise) and is refused with blockwise scales.
    out_dtype torch.float8_e4m3fn or torch.float8_e5m2 writes FP8: out = fp8(v / scale_result), v the fp32 value the
    other outputs round, fp8() round to nearest with finite values saturated to the format's largest (b200_gemm_fp8_q8 /
    b200_gemm_fp8_blockwise_q8, static mode).  scale_result is None (1) or a one-element float32 CUDA tensor, read on the
    device; the bias is then bf16.  Every input recipe above works with an FP8 out_dtype.
    Operands of other dtypes, or two e5m2 operands, are a TypeError; a scale of another shape or dtype, a CPU tensor,
    another bias, out_dtype, scale_result or out (shape, dtype, or rows that overlap) is a ValueError."""
    import torch
    out_dtype = out_dtype or (out.dtype if out is not None else torch.bfloat16)
    if _is_fp8(out_dtype):
        return _scaled_mm_fp8_out(A, B, scale_a, scale_b, bias, None, out_dtype, use_fast_accum, out, None, scale_result,
                                  stream)[0]
    if scale_result is not None:
        raise ValueError("scale_result applies to an FP8 out_dtype only")
    ta, tb, m, n, k, op_a, lda, op_b, ldb, rows, blocks = _scaled_mm_args(A, B, scale_a, scale_b, bias, out_dtype,
                                                                          use_fast_accum, out, fp8_out=False)
    if out is None:
        out = torch.empty((m, n), dtype=out_dtype, device=A.device)
    if m == 0 or n == 0:
        return out
    ot = {torch.float32: OUT_F32, torch.bfloat16: OUT_BF16, torch.float16: OUT_F16}[out_dtype]
    if blocks is not None:
        _check(lib.b200_gemm_fp8_blockwise(op_a, op_b, ta, tb, m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb,
                                           scale_a.data_ptr(), blocks[0], scale_a.stride(0), scale_a.stride(1),
                                           scale_b.data_ptr(), blocks[1], scale_b.stride(0), scale_b.stride(1),
                                           bias.data_ptr() if bias is not None else None, out.data_ptr(), _ld(out), ot,
                                           _stream_ptr(stream)))
        return out
    _check(lib.b200_gemm_fp8(op_a, op_b, ta, tb, m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb, scale_a.data_ptr(),
                             rows[0], scale_b.data_ptr(), rows[1], bias.data_ptr() if bias is not None else None,
                             out.data_ptr(), _ld(out), ot, int(bool(use_fast_accum)), _stream_ptr(stream)))
    return out


def _resolve_scales(scale_a, scale_b, m, n, k):
    """(rows, blocks) of scaled_mm's scale resolution: rows = (scale_a_rowwise, scale_b_colwise) for tensorwise /
    rowwise scales, else blocks = (scale_a_block, scale_b_block); a ValueError when neither fits."""
    import torch
    rows = []
    for name, s, length, shape in (("scale_a", scale_a, m, (m, 1)), ("scale_b", scale_b, n, (1, n))):
        if s.dtype != torch.float32:
            raise ValueError(f"{name} must be float32, not {s.dtype}")
        if s.numel() == 1:
            rows.append(0)
        elif s.numel() == length and tuple(s.shape) == shape and s.is_contiguous():
            rows.append(1)
        else:
            rows = None
            break
    blocks = _blockwise_recipe(scale_a, scale_b, m, n, k) if rows is None else None
    if rows is None and blocks is None:
        q = -(-k // 128)
        raise ValueError(f"scale_a and scale_b must have one element, shapes (m, 1) and (1, n), or blockwise shapes "
                         f"(({m}, {q}), ({q}, {-(-n // 128)})), (({m}, {q}), ({q}, {n})) or "
                         f"(({-(-m // 128)}, {q}), ({q}, {n})), not {tuple(scale_a.shape)} and {tuple(scale_b.shape)}")
    return rows, blocks


def _scaled_mm_args(A, B, scale_a, scale_b, bias, out_dtype, use_fast_accum, out, fp8_out, activation=None,
                    scale_result=None, out_scale=None):
    """scaled_mm's operand, shape and scale resolution and its refusals, in its order, for a 16-bit / fp32 (fp8_out
    False) or an FP8 out_dtype (with scaled_mm_quant's activation and out_scale, and scale_result); returns
    (ta, tb, m, n, k, op_a, lda, op_b, ldb, rows, blocks), rows and blocks as _resolve_scales gives them."""
    import torch
    ta, tb = _fp8_type(A), _fp8_type(B)
    if ta is None or tb is None:
        raise TypeError(f"operands must be float8_e4m3fn or float8_e5m2, not {A.dtype} and {B.dtype}")
    if ta == FP8_E5M2 and tb == FP8_E5M2:
        raise TypeError("float8_e5m2 x float8_e5m2 is not supported (as in torch._scaled_mm)")
    if A.dim() != 2 or B.dim() != 2 or A.shape[1] != B.shape[0]:
        raise ValueError(f"A and B must be 2-D with matching inner dimensions, not {tuple(A.shape)} and {tuple(B.shape)}")
    m, k = A.shape
    n = B.shape[1]
    if fp8_out and not _is_fp8(out_dtype):
        raise ValueError(f"out_dtype must be float8_e4m3fn or float8_e5m2, not {out_dtype}")
    if not fp8_out and out_dtype not in (torch.bfloat16, torch.float16, torch.float32):
        raise ValueError(f"out_dtype must be bfloat16, float16 or float32, not {out_dtype}")
    if fp8_out and activation not in ACTIVATIONS:
        raise ValueError(f"activation must be one of {sorted(a for a in ACTIVATIONS if a)} or None, not {activation!r}")
    rows, blocks = _resolve_scales(scale_a, scale_b, m, n, k)
    if blocks is not None and use_fast_accum:
        raise ValueError("use_fast_accum=True is not available with blockwise scales: their scales change every k-block")
    if bias is not None:
        if fp8_out and bias.dtype != torch.bfloat16:
            raise ValueError(f"with an FP8 output the bias must be bfloat16, not {bias.dtype}")
        if not fp8_out and bias.dtype != out_dtype:
            raise ValueError(f"the bias must have dtype {out_dtype}, not {bias.dtype}")
        if bias.dim() != 1 or bias.shape[0] != n or not bias.is_contiguous():
            raise ValueError(f"the bias must be contiguous and 1-D with n = {n} elements, not of shape {tuple(bias.shape)}")
    if scale_result is not None and (scale_result.dtype != torch.float32 or scale_result.numel() != 1):
        raise ValueError(f"scale_result must be one float32 element, not {scale_result.dtype} of shape "
                         f"{tuple(scale_result.shape)}")
    if out is not None:
        if out.dtype != out_dtype or tuple(out.shape) != (m, n):
            raise ValueError(f"out must be {out_dtype} of shape {(m, n)}, not {out.dtype} of shape {tuple(out.shape)}")
        if (n > 1 and out.stride(1) != 1) or (m > 1 and out.stride(0) < n):
            raise ValueError(f"out must be row-major with rows that do not overlap, not of strides {tuple(out.stride())}")
    qn = -(-n // 128)
    if out_scale is not None:
        if out_scale.dtype != torch.float32 or tuple(out_scale.shape) != (m, qn):
            raise ValueError(f"out_scale must be float32 of shape {(m, qn)}, not {out_scale.dtype} of shape "
                             f"{tuple(out_scale.shape)}")
        sr_, sb_ = out_scale.stride()
        row_major = (qn == 1 or sb_ == 1) and (m == 1 or sr_ >= qn)
        col_major = (m == 1 or sr_ == 1) and (qn == 1 or sb_ >= m)
        if not (row_major or col_major):
            raise ValueError(f"out_scale must be row-major or outer-dim-major without overlap, not of strides "
                             f"{tuple(out_scale.stride())}")
    op_a, lda = operand_layout(tuple(A.shape), A.stride())
    op_b, ldb = operand_layout(tuple(B.shape), B.stride())
    tensors = [A, B, scale_a, scale_b] + [t for t in (bias, out, out_scale, scale_result) if t is not None]
    if not all(t.is_cuda for t in tensors):
        raise ValueError("A, B, the scales, the bias, scale_result, out and out_scale must be CUDA tensors" if fp8_out
                         else "A, B, the scales, the bias and out must be CUDA tensors")
    return ta, tb, m, n, k, op_a, lda, op_b, ldb, rows, blocks


def _scaled_mm_fp8_out(A, B, scale_a, scale_b, bias, activation, out_dtype, use_fast_accum, out, out_scale,
                       scale_result, stream, dynamic=False):
    """The FP8-output form of scaled_mm (static: scale_result) and scaled_mm_quant (dynamic: out_scale); returns
    (out, scale_c or None).  Every check happens before the device is touched."""
    import torch
    ta, tb, m, n, k, op_a, lda, op_b, ldb, rows, blocks = _scaled_mm_args(
        A, B, scale_a, scale_b, bias, out_dtype, use_fast_accum, out, fp8_out=True, activation=activation,
        scale_result=scale_result, out_scale=out_scale)
    if out is None:
        out = torch.empty((m, n), dtype=out_dtype, device=A.device)
    if dynamic and out_scale is None:
        out_scale = torch.empty((m, -(-n // 128)), dtype=torch.float32, device=A.device)
    if m == 0 or n == 0:
        return out, out_scale
    ct = FP8_E4M3 if out_dtype == torch.float8_e4m3fn else FP8_E5M2
    act = ACTIVATIONS[activation]
    bi = bias.data_ptr() if bias is not None else None
    sr = scale_result.data_ptr() if scale_result is not None else None
    sc, sc_row, sc_blk = (out_scale.data_ptr(), *out_scale.stride()) if dynamic else (None, 0, 0)
    if blocks is not None:
        _check(lib.b200_gemm_fp8_blockwise_q8(op_a, op_b, ta, tb, m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb,
                                              scale_a.data_ptr(), blocks[0], scale_a.stride(0), scale_a.stride(1),
                                              scale_b.data_ptr(), blocks[1], scale_b.stride(0), scale_b.stride(1), bi,
                                              act, ct, out.data_ptr(), _ld(out), sr, sc, sc_row, sc_blk,
                                              _stream_ptr(stream)))
    else:
        _check(lib.b200_gemm_fp8_q8(op_a, op_b, ta, tb, m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb, scale_a.data_ptr(),
                                    rows[0], scale_b.data_ptr(), rows[1], bi, act, int(bool(use_fast_accum)), ct,
                                    out.data_ptr(), _ld(out), sr, sc, sc_row, sc_blk, _stream_ptr(stream)))
    return out, out_scale


def scaled_mm_quant(A, B, scale_a, scale_b, bias=None, activation=None, out_dtype=None, use_fast_accum=False,
                    out=None, out_scale=None, stream=None):
    """scaled_mm with a fused 1 x 128 quantisation of its output: returns (C, scale_c) with C FP8 (out_dtype
    torch.float8_e4m3fn, the default, or torch.float8_e5m2) and scale_c float32 (m, ceil(n / 128)), so that
    C[i, j] * scale_c[i, j // 128] ~ act(A @ B * scales + bias)[i, j] (b200_gemm_fp8_q8 / b200_gemm_fp8_blockwise_q8,
    dynamic mode).  Per row and 128-column block, d = amax / F (F = 448 or 57344; 1 for an all-zero block, NaN for a
    block holding a NaN or an inf) and C = fp8(v / d).  (C, scale_c) is the (A, scale_a) of a following 1 x 128
    blockwise scaled_mm: scaled_mm(C, W2.t(), scale_c, sW2) runs the next layer with no conversion in between.
    A, B, scale_a, scale_b and use_fast_accum are scaled_mm's; bias is None or n contiguous bf16 values; activation
    takes gemm()'s strings (None, "relu", "gelu", "gelu_tanh").  out_scale may be any (m, ceil(n / 128)) float32 view
    that is row-major or outer-dim-major (torch's layout for scale_a); a new one is row-major.  The refusals are
    scaled_mm's, and an out_scale of another shape, dtype or layout is a ValueError."""
    import torch
    out_dtype = out_dtype or (out.dtype if out is not None else torch.float8_e4m3fn)
    return _scaled_mm_fp8_out(A, B, scale_a, scale_b, bias, activation, out_dtype, use_fast_accum, out, out_scale, None,
                              stream, dynamic=True)


def _fp8_in_place(name, t, ld, entry_stride, entry_elems):
    """Refuses (ValueError) an FP8 operand the tensor cores cannot read in place: a base or a pitch that is not a
    multiple of 16 bytes, or an entry stride other than 0 or a 16-byte multiple of at least one entry."""
    if t.data_ptr() % 16 or ld % 16:
        raise ValueError(f"{name} must have a 16-byte aligned base and a pitch that is a multiple of 16 bytes "
                         f"(pitch {ld})")
    if entry_stride != 0 and (entry_stride % 16 or entry_stride < entry_elems):
        raise ValueError(f"{name}'s stride(0) must be 0 or a multiple of 16 bytes of at least one entry "
                         f"({entry_elems} elements), not {entry_stride}")


def _grouped_blockwise_recipe(A, scale_a, scale_b, groups, n, k):
    """(scale_a_block, scale_b_block) of a grouped (2-D A) or batched (3-D A) blockwise call, resolved from the
    scales' shapes in scaled_mm's order, or None.  scale_b is (G, q, ceil(n / 128)) or (G, q, n); scale_a is
    (total_m, q) for a 2-D A (1 x 128 only), and (G, m, q) or (G, ceil(m / 128), q) for a 3-D A."""
    q, nb = -(-k // 128), -(-n // 128)
    if A.dim() == 2:
        want_a = {1: (A.shape[0], q)}
    else:
        m = A.shape[1]
        want_a = {1: (groups, m, q), 128: (groups, -(-m // 128), q)}
    want_b = {128: (groups, q, nb), 1: (groups, q, n)}
    for blocks in ((1, 128), (1, 1), (128, 1)):
        if blocks[0] in want_a and tuple(scale_a.shape) == want_a[blocks[0]] and tuple(scale_b.shape) == want_b[blocks[1]]:
            return blocks
    return None


def scaled_grouped_mm(A, B, scale_a, scale_b, offs=None, out_dtype=None, use_fast_accum=False, out=None, stream=None):
    """torch._scaled_grouped_mm for FP8 mixture-of-experts layers: every group, or every entry of a batch, is one
    scaled_mm with rowwise scales, all of them in one launch (b200_gemm_fp8_grouped / _batched), or with blockwise
    scales one blockwise scaled_mm (b200_gemm_fp8_blockwise_grouped / _batched).

    B is 3-D (G, k, n) and column-major in its last two dimensions: W.transpose(-2, -1) of a (G, n, k) weight, read
    in place.  scale_b is float32 (G, n), contiguous along n.  Then either
      A 2-D (total_m, k) row-major, scale_a (total_m,) contiguous, and offs a contiguous 1-D int32 CUDA tensor of G
        cumulative end rows: rows [offs[g-1], offs[g]) of out are (A[rows] @ B[g]) * scale_a[rows, None] * scale_b[g],
        with the offsets clamped as in gemm(offs=...) and read on the device; rows from offs[-1] on are not written (a
        new out is torch.empty there, as in torch);
      A 3-D (G, m, k) row-major in its last two dimensions (an expand()ed A is broadcast), scale_a (G, m) contiguous
        along m, and no offs: out[g] = (A[g] @ B[g]) * scale_a[g, :, None] * scale_b[g].
    Blockwise scales (DeepSeek-V3's recipe), with q = ceil(k / 128): a 3-D scale_b, (G, q, ceil(n / 128)) for 128 x 128
    weight blocks or (G, q, n) for 1 x 128, with scale_a (total_m, q) for a 2-D A (1 x 128 only: a 128-row block
    would straddle groups), or (G, m, q) or (G, ceil(m / 128), q) for a 3-D A; the pair of 128 x 128 shapes is
    refused.  Scales are float32 CUDA tensors of any strides (torch's outer-dim-major layout is read in place).  A
    shape that fits two recipes resolves in scaled_mm's order, which gives the same result.  Each group or entry is
    then the blockwise scaled_mm without bias on its rows, B and scales; use_fast_accum=True is refused.
    Each step is rounded as in scaled_mm, so each group or entry is bit for bit scaled_mm on its own rows, B and
    scales.  Operands are float8_e4m3fn or float8_e5m2 (not both e5m2).  out_dtype is torch.bfloat16 (the default, as
    in torch), torch.float16 or torch.float32.  use_fast_accum as in scaled_mm.  The offsets and scales stay on the
    device: the call never synchronises and can be captured in a CUDA graph.
    Operands of other dtypes are a TypeError.  A 2-D B (torch's 2-D x 2-D and 3-D x 2-D forms), another layout, an
    operand the tensor cores cannot read in place (16-byte aligned bases and pitches, entry strides 0 or at least one
    entry), another scale, offs, out_dtype or out, or a CPU tensor is a ValueError."""
    import torch
    out_dtype = out_dtype or (out.dtype if out is not None else torch.bfloat16)
    g = _scaled_grouped_args(A, B, scale_a, scale_b, offs, out_dtype, use_fast_accum, out, fp8_out=False)
    tensors = [A, B, scale_a, scale_b] + [t for t in (offs, out) if t is not None]
    if not all(t.is_cuda for t in tensors):
        raise ValueError("A, B, the scales, offs and out must be CUDA tensors")
    if out is None:
        out = torch.empty(g.shape, dtype=out_dtype, device=A.device)
    if g.groups == 0 or out.numel() == 0:
        return out
    g.check_in_place(A, B)
    ta, tb, groups, n, k, lda, ldb, sb, ssb, blocks = g.ta, g.tb, g.groups, g.n, g.k, g.lda, g.ldb, g.sb, g.ssb, g.blocks
    ot = {torch.float32: OUT_F32, torch.bfloat16: OUT_BF16, torch.float16: OUT_F16}[out_dtype]
    fast = int(bool(use_fast_accum))
    if blocks is not None and A.dim() == 2:
        _check(lib.b200_gemm_fp8_blockwise_grouped(ta, tb, g.m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb, sb,
                                                   offs.data_ptr(), groups, scale_a.data_ptr(), scale_a.stride(0),
                                                   scale_a.stride(1), scale_b.data_ptr(), blocks[1], scale_b.stride(1),
                                                   scale_b.stride(2), ssb, out.data_ptr(), _ld(out), ot,
                                                   _stream_ptr(stream)))
    elif blocks is not None:
        _check(lib.b200_gemm_fp8_blockwise_batched(ta, tb, g.m, n, k, A.data_ptr(), lda, A.stride(0) if groups > 1 else 0,
                                                   B.data_ptr(), ldb, sb, scale_a.data_ptr(), blocks[0],
                                                   scale_a.stride(1), scale_a.stride(2),
                                                   scale_a.stride(0) if groups > 1 else 0, scale_b.data_ptr(), blocks[1],
                                                   scale_b.stride(1), scale_b.stride(2), ssb, out.data_ptr(),
                                                   _ld(out[0]), out.stride(0) if groups > 1 else 0, groups, ot,
                                                   _stream_ptr(stream)))
    elif A.dim() == 2:
        _check(lib.b200_gemm_fp8_grouped(ta, tb, g.m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb, sb,
                                         offs.data_ptr(), groups, scale_a.data_ptr(), scale_b.data_ptr(), ssb,
                                         out.data_ptr(), _ld(out), ot, fast, _stream_ptr(stream)))
    else:
        _check(lib.b200_gemm_fp8_batched(ta, tb, g.m, n, k, A.data_ptr(), lda, A.stride(0) if groups > 1 else 0,
                                         B.data_ptr(), ldb, sb, scale_a.data_ptr(),
                                         scale_a.stride(0) if groups > 1 else 0, scale_b.data_ptr(), ssb,
                                         out.data_ptr(), _ld(out[0]), out.stride(0) if groups > 1 else 0, groups, ot,
                                         fast, _stream_ptr(stream)))
    return out


class _GroupedArgs:
    """The operands of a scaled_grouped_mm / scaled_grouped_mm_quant call as the C ABI reads them."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def check_in_place(self, A, B):
        if self.k > 0:
            _fp8_in_place("A", A, self.lda, A.stride(0) if A.dim() == 3 and self.groups > 1 else 0, A.shape[-2] * self.lda)
            _fp8_in_place("B", B, self.ldb, self.sb, self.n * self.ldb)


def _scaled_grouped_args(A, B, scale_a, scale_b, offs, out_dtype, use_fast_accum, out, fp8_out):
    """scaled_grouped_mm's shape resolution and refusals, in its order, for a 16-bit / fp32 (fp8_out False) or an FP8
    out_dtype; every check but the operands' in-place rule (check_in_place), which applies only with work to do, and
    the callers' check that every tensor is on the GPU."""
    import torch
    ta, tb = _fp8_type(A), _fp8_type(B)
    if ta is None or tb is None:
        raise TypeError(f"operands must be float8_e4m3fn or float8_e5m2, not {A.dtype} and {B.dtype}")
    if ta == FP8_E5M2 and tb == FP8_E5M2:
        raise TypeError("float8_e5m2 x float8_e5m2 is not supported (as in torch._scaled_mm)")
    if B.dim() == 2 and A.dim() in (2, 3):
        raise ValueError(f"the {A.dim()}-D x 2-D form of torch._scaled_grouped_mm is not supported: B must be 3-D")
    if A.dim() not in (2, 3) or B.dim() != 3:
        raise ValueError(f"A must be 2-D or 3-D and B 3-D, not {A.dim()}-D and {B.dim()}-D")
    groups, k, n = B.shape
    if A.shape[-1] != k:
        raise ValueError(f"contraction dimensions differ: A is {tuple(A.shape)}, B is {tuple(B.shape)}")
    if fp8_out and not _is_fp8(out_dtype):
        raise ValueError(f"out_dtype must be float8_e4m3fn or float8_e5m2, not {out_dtype}")
    if not fp8_out and out_dtype not in (torch.bfloat16, torch.float16, torch.float32):
        raise ValueError(f"out_dtype must be bfloat16, float16 or float32, not {out_dtype}")
    try:
        op_a, lda = operand_layout(tuple(A.shape[-2:]), A.stride()[-2:])
        op_bt, ldb = operand_layout((n, k), (B.stride(2), B.stride(1)))      # B_g^T (n x k) must be row-major
    except ValueError as e:
        raise ValueError(f"A must be row-major and B column-major in their last two dimensions: {e}") from None
    if op_a != OP_N or op_bt != OP_N:
        raise ValueError(f"A must be row-major and B column-major in their last two dimensions, not of strides "
                         f"{tuple(A.stride())} and {tuple(B.stride())}")
    sb = B.stride(0) if groups > 1 else 0
    for name, s in (("scale_a", scale_a), ("scale_b", scale_b)):
        if s.dtype != torch.float32:
            raise ValueError(f"{name} must be float32, not {s.dtype}")
    if scale_b.dim() == 3:
        q, mq = -(-k // 128), "total_m" if A.dim() == 2 else "m or ceil(m / 128)"
        if _grouped_blockwise_recipe(A, scale_a, scale_b, groups, n, k) is None:
            raise ValueError(f"blockwise scales must be scale_b ({groups}, {q}, {-(-n // 128)}) or ({groups}, {q}, {n}) "
                             f"with scale_a ({mq}, {q}) (not both 128 x 128), not {tuple(scale_a.shape)} and "
                             f"{tuple(scale_b.shape)}")
    elif scale_b.dim() != 2 or tuple(scale_b.shape) != (groups, n) or (n > 1 and scale_b.stride(1) != 1):
        raise ValueError(f"scale_b must be ({groups}, {n}) and contiguous along n, not {tuple(scale_b.shape)} of "
                         f"strides {tuple(scale_b.stride())}")
    ssb = scale_b.stride(0) if groups > 1 else 0
    blocks = _grouped_blockwise_recipe(A, scale_a, scale_b, groups, n, k) if scale_b.dim() == 3 else None
    if blocks is not None and use_fast_accum:
        raise ValueError("use_fast_accum=True is not available with blockwise scales: their scales change every k-block")
    if A.dim() == 2:
        if offs is None:
            raise ValueError("a 2-D A needs offs, the groups' cumulative end rows")
        _check_offs(offs)
        if offs.numel() != groups:
            raise ValueError(f"offs has {offs.numel()} elements for {groups} groups of B")
        if groups > 1 and sb < n * ldb:
            raise ValueError(f"the groups of B must not overlap or be broadcast (stride(0) = {B.stride(0)})")
        m = A.shape[0]
        if blocks is None and (scale_a.dim() != 1 or scale_a.shape[0] != m or not scale_a.is_contiguous()):
            raise ValueError(f"scale_a must be contiguous and 1-D with {m} elements, not {tuple(scale_a.shape)}")
        shape = (m, n)
    else:
        if offs is not None:
            raise ValueError("offs must be None for a 3-D A: every entry has its own rows")
        if A.shape[0] != groups:
            raise ValueError(f"batch sizes differ: {A.shape[0]} and {groups}")
        m = A.shape[1]
        if blocks is None and (scale_a.dim() != 2 or tuple(scale_a.shape) != (groups, m) or (m > 1 and scale_a.stride(1) != 1)):
            raise ValueError(f"scale_a must be ({groups}, {m}) and contiguous along m, not {tuple(scale_a.shape)} of "
                             f"strides {tuple(scale_a.stride())}")
        shape = (groups, m, n)
    if out is not None:
        if out.dtype != out_dtype or tuple(out.shape) != shape:
            raise ValueError(f"out must be {out_dtype} of shape {shape}, not {out.dtype} of shape {tuple(out.shape)}")
        rows, cols = shape[-2:]
        if (cols > 1 and out.stride(-1) != 1) or (rows > 1 and out.stride(-2) < cols):
            raise ValueError(f"out must be row-major with rows that do not overlap, not of strides {tuple(out.stride())}")
        if len(shape) == 3 and groups > 1 and rows * cols > 0 and out.stride(0) < (rows - 1) * out.stride(1) + cols:
            raise ValueError(f"the entries of out must not overlap (stride(0) = {out.stride(0)})")
    return _GroupedArgs(ta=ta, tb=tb, groups=groups, m=m, n=n, k=k, lda=lda, ldb=ldb, sb=sb, ssb=ssb, blocks=blocks,
                        shape=shape)


def scaled_grouped_mm_quant(A, B, scale_a, scale_b, offs=None, activation=None, out_dtype=None, use_fast_accum=False,
                            out=None, out_scale=None, stream=None):
    """scaled_grouped_mm with a fused 1 x 128 quantisation of every group's or entry's output: returns (C, scale_c)
    with C FP8 (out_dtype torch.float8_e4m3fn, the default, or torch.float8_e5m2) and scale_c float32, (total_m,
    ceil(n / 128)) for a 2-D A and (G, m, ceil(n / 128)) for a 3-D A (b200_gemm_fp8_grouped_q8 / _batched_q8 /
    _blockwise_grouped_q8 / _blockwise_batched_q8).  Each group or entry is bit for bit scaled_mm_quant on its own
    rows, B and scales without bias: per row and 128-column block d = amax / F (F = 448 or 57344; 1 for an all-zero
    block, NaN for a block holding a NaN or an inf) and C = fp8(v / d), v = act(the fp32 value scaled_grouped_mm rounds).
    A 2-D A's scale_c is indexed by the row of C, so scaled_grouped_mm(C, W2.transpose(-2, -1), scale_c, sW2, offs)
    runs the next layer with no conversion; rows from offs[-1] on are written in neither.
    A, B, scale_a, scale_b, offs, use_fast_accum, out and the refusals are scaled_grouped_mm's; activation takes
    gemm()'s strings (None, "relu", "gelu", "gelu_tanh").  out_scale may be any float32 view of scale_c's shape whose
    last two dimensions are row-major or outer-dim-major (for a 3-D A, entries that do not overlap); a new one is
    row-major.  Another out_scale or activation is a ValueError."""
    import torch
    out_dtype = out_dtype or (out.dtype if out is not None else torch.float8_e4m3fn)
    if activation not in ACTIVATIONS:
        raise ValueError(f"activation must be one of {sorted(a for a in ACTIVATIONS if a)} or None, not {activation!r}")
    g = _scaled_grouped_args(A, B, scale_a, scale_b, offs, out_dtype, use_fast_accum, out, fp8_out=True)
    groups, n, k = g.groups, g.n, g.k
    qn = -(-n // 128)
    sc_shape = g.shape[:-1] + (qn,)
    if out_scale is not None:
        if out_scale.dtype != torch.float32 or tuple(out_scale.shape) != sc_shape:
            raise ValueError(f"out_scale must be float32 of shape {sc_shape}, not {out_scale.dtype} of shape "
                             f"{tuple(out_scale.shape)}")
        rows = sc_shape[-2]
        sr_, sb_ = out_scale.stride()[-2:]
        row_major = (qn == 1 or sb_ == 1) and (rows == 1 or sr_ >= qn)
        col_major = (rows == 1 or sr_ == 1) and (qn == 1 or sb_ >= rows)
        if not (row_major or col_major):
            raise ValueError(f"out_scale must be row-major or outer-dim-major without overlap in its last two "
                             f"dimensions, not of strides {tuple(out_scale.stride())}")
        if (len(sc_shape) == 3 and groups > 1 and rows * qn > 0 and
                out_scale.stride(0) < (rows - 1) * sr_ + (qn - 1) * sb_ + 1):
            raise ValueError(f"the entries of out_scale must not overlap (stride(0) = {out_scale.stride(0)})")
    tensors = [A, B, scale_a, scale_b] + [t for t in (offs, out, out_scale) if t is not None]
    if not all(t.is_cuda for t in tensors):
        raise ValueError("A, B, the scales, offs, out and out_scale must be CUDA tensors")
    if out is None:
        out = torch.empty(g.shape, dtype=out_dtype, device=A.device)
    if out_scale is None:
        out_scale = torch.empty(sc_shape, dtype=torch.float32, device=A.device)
    if groups == 0 or out.numel() == 0:
        return out, out_scale
    g.check_in_place(A, B)
    ta, tb, lda, ldb, sb, ssb, blocks = g.ta, g.tb, g.lda, g.ldb, g.sb, g.ssb, g.blocks
    ct = FP8_E4M3 if out_dtype == torch.float8_e4m3fn else FP8_E5M2
    act = ACTIVATIONS[activation]
    fast = int(bool(use_fast_accum))
    sc_row, sc_blk = out_scale.stride()[-2:]
    st = _stream_ptr(stream)
    if A.dim() == 2:
        if blocks is not None:
            _check(lib.b200_gemm_fp8_blockwise_grouped_q8(
                ta, tb, g.m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb, sb, offs.data_ptr(), groups, scale_a.data_ptr(),
                scale_a.stride(0), scale_a.stride(1), scale_b.data_ptr(), blocks[1], scale_b.stride(1), scale_b.stride(2),
                ssb, act, ct, out.data_ptr(), _ld(out), out_scale.data_ptr(), sc_row, sc_blk, st))
        else:
            _check(lib.b200_gemm_fp8_grouped_q8(ta, tb, g.m, n, k, A.data_ptr(), lda, B.data_ptr(), ldb, sb,
                                                offs.data_ptr(), groups, scale_a.data_ptr(), scale_b.data_ptr(), ssb, act,
                                                fast, ct, out.data_ptr(), _ld(out), out_scale.data_ptr(), sc_row, sc_blk,
                                                st))
        return out, out_scale
    sa_e, c_e, sc_e = ((A.stride(0), out.stride(0), out_scale.stride(0)) if groups > 1 else (0, 0, 0))
    if blocks is not None:
        _check(lib.b200_gemm_fp8_blockwise_batched_q8(
            ta, tb, g.m, n, k, A.data_ptr(), lda, sa_e, B.data_ptr(), ldb, sb, scale_a.data_ptr(), blocks[0],
            scale_a.stride(1), scale_a.stride(2), scale_a.stride(0) if groups > 1 else 0, scale_b.data_ptr(), blocks[1],
            scale_b.stride(1), scale_b.stride(2), ssb, act, ct, out.data_ptr(), _ld(out[0]), c_e, out_scale.data_ptr(),
            sc_row, sc_blk, sc_e, groups, st))
    else:
        _check(lib.b200_gemm_fp8_batched_q8(ta, tb, g.m, n, k, A.data_ptr(), lda, sa_e, B.data_ptr(), ldb, sb,
                                            scale_a.data_ptr(), scale_a.stride(0) if groups > 1 else 0,
                                            scale_b.data_ptr(), ssb, act, fast, ct, out.data_ptr(), _ld(out[0]), c_e,
                                            out_scale.data_ptr(), sc_row, sc_blk, sc_e, groups, st))
    return out, out_scale


def _scale_layout_ok(rows, blks, s_row, s_blk):
    """b200_gemm_fp8_q8's rule for a scale matrix: row-major or outer-dim-major, an extent-1 dimension's stride free."""
    row_major = (blks == 1 or s_blk == 1) and (rows == 1 or s_row >= blks)
    col_major = (rows == 1 or s_row == 1) and (blks == 1 or s_blk >= rows)
    return row_major or col_major


def quantize_fp8(x, block=(1, 128), dtype=None, transpose=False, out=None, out_scale=None, stream=None):
    """Blockwise FP8 quantisation of x on the device (b200_fp8_quantize): returns (q, s), or (q, s, qt, st) with
    transpose=True, the operands and scales that scaled_mm / scaled_grouped_mm take with blockwise scales.

    x is a 2-D (m, k) or 3-D (G, m, k) CUDA tensor of bfloat16, float16 or float32 with unit last stride, rows at any
    pitch.  dtype is torch.float8_e4m3fn (the default, F = 448) or torch.float8_e5m2 (F = 57344).  For each block,
    d = amax / F (amax the largest |x| in the block; 1 for an all-zero block, NaN for a block holding a NaN or an inf)
    and q = fp8(x / d), rounded to nearest even with finite values saturated to +-F: the rule of scaled_mm_quant's
    epilogue, bit for bit.  block is
      (1, 128)    activations and gradients: s (..., m, ceil(k / 128)), one scale per row and 128 columns.  qt (..., k,
                  m) is the (1, 128) quantisation of x^T, with st (..., k, ceil(m / 128)): x's 128 x 1 blocks.
      (128, 128)  weights: s (..., ceil(m / 128), ceil(k / 128)).  qt is q^T byte for byte and st = s.transpose(-2, -1),
                  a view of s.
    q and qt are written in one launch that reads x once.  A blockwise FP8 linear layer y = x @ W.t() (W is (n, k)):
      xq, xs, xqt, xst = quantize_fp8(x, transpose=True)
      wq, ws, wqt, _ = quantize_fp8(W, block=(128, 128), transpose=True)
      dyq, dys, dyqt, dyst = quantize_fp8(dy, transpose=True)
      y  = scaled_mm(xq, wq.t(), xs, ws.t())             # forward
      dx = scaled_mm(dyq, wqt.t(), dys, ws)              # dgrad: dy @ W
      dw = scaled_mm(dyqt, xqt.t(), dyst, xst.t())       # wgrad: dy^T @ x, 128 x 1 blocks along the tokens
    and a mixture-of-experts layer with expert weights W (G, n, k) and tokens grouped by offs:
      wq, ws, wqt, _ = quantize_fp8(W, block=(128, 128), transpose=True)
      y  = scaled_grouped_mm(xq, wq.transpose(-2, -1), xs, ws.transpose(-2, -1), offs)   # forward
      dx = scaled_grouped_mm(dyq, wqt.transpose(-2, -1), dys, ws, offs)                 # dgrad
    out (q) may be any FP8 tensor of x's shape and dtype whose rows (and entries) do not overlap; out_scale any float32
    tensor of s's shape that is row-major or outer-dim-major in its last two dimensions (torch's layout for scale_a),
    entries not overlapping.  New tensors are row-major.  The call never synchronises and can be captured in a CUDA graph.
    An input or dtype of another type is a TypeError; another block, shape, layout, out or out_scale, or a CPU tensor, is
    a ValueError."""
    import torch
    dtype = dtype or (out.dtype if out is not None else torch.float8_e4m3fn)
    in_type = {torch.float32: OUT_F32, torch.bfloat16: OUT_BF16, torch.float16: OUT_F16}.get(x.dtype)
    if in_type is None:
        raise TypeError(f"x must be bfloat16, float16 or float32, not {x.dtype}")
    if not _is_fp8(dtype):
        raise TypeError(f"dtype must be float8_e4m3fn or float8_e5m2, not {dtype}")
    block = tuple(block)
    if block not in ((1, 128), (128, 128)):
        raise ValueError(f"block must be (1, 128) or (128, 128), not {block}")
    if x.dim() not in (2, 3):
        raise ValueError(f"x must be 2-D or 3-D, not {x.dim()}-D")
    lead, (m, k) = tuple(x.shape[:-2]), tuple(x.shape[-2:])
    groups = lead[0] if lead else 1
    if k > 1 and x.stride(-1) != 1:
        raise ValueError(f"x must have a unit last stride, not strides {tuple(x.stride())}")
    if m > 1 and x.stride(-2) < k:
        raise ValueError(f"x's rows must not overlap: stride(-2) = {x.stride(-2)} < {k}")
    qm, qk = -(-m // 128), -(-k // 128)
    s_shape = lead + ((m if block[0] == 1 else qm), qk)
    if out is not None:
        if out.dtype != dtype or tuple(out.shape) != tuple(x.shape):
            raise ValueError(f"out must be {dtype} of shape {tuple(x.shape)}, not {out.dtype} of shape {tuple(out.shape)}")
        if (k > 1 and out.stride(-1) != 1) or (m > 1 and out.stride(-2) < k):
            raise ValueError(f"out must be row-major with rows that do not overlap, not of strides {tuple(out.stride())}")
        if lead and groups > 1 and m * k > 0 and out.stride(0) < (m - 1) * out.stride(-2) + k:
            raise ValueError(f"the entries of out must not overlap (stride(0) = {out.stride(0)})")
    if out_scale is not None:
        if out_scale.dtype != torch.float32 or tuple(out_scale.shape) != s_shape:
            raise ValueError(f"out_scale must be float32 of shape {s_shape}, not {out_scale.dtype} of shape "
                             f"{tuple(out_scale.shape)}")
        rows, blks = s_shape[-2:]
        sr_, sb_ = out_scale.stride()[-2:]
        if not _scale_layout_ok(rows, blks, sr_, sb_):
            raise ValueError(f"out_scale must be row-major or outer-dim-major without overlap in its last two "
                             f"dimensions, not of strides {tuple(out_scale.stride())}")
        if lead and groups > 1 and rows * blks > 0 and out_scale.stride(0) < (rows - 1) * sr_ + (blks - 1) * sb_ + 1:
            raise ValueError(f"the entries of out_scale must not overlap (stride(0) = {out_scale.stride(0)})")
    if not all(t.is_cuda for t in (x, out, out_scale) if t is not None):
        raise ValueError("x, out and out_scale must be CUDA tensors")
    q = out if out is not None else torch.empty(x.shape, dtype=dtype, device=x.device)
    s = out_scale if out_scale is not None else torch.empty(s_shape, dtype=torch.float32, device=x.device)
    qt = st = None
    if transpose:
        qt = torch.empty(lead + (k, m), dtype=dtype, device=x.device)
        st = torch.empty(lead + (k, qm), dtype=torch.float32, device=x.device) if block[0] == 1 else s.transpose(-2, -1)
    if x.numel() > 0:
        e = (lambda t: t.stride(0) if lead and groups > 1 else 0)
        ld = (lambda t: t.stride(-2) if t.shape[-2] > 1 else t.shape[-1])
        ct = FP8_E4M3 if dtype == torch.float8_e4m3fn else FP8_E5M2
        t_args = (qt.data_ptr(), ld(qt), e(qt)) if transpose else (None, 0, 0)
        st_args = (st.data_ptr(), *st.stride()[-2:], e(st)) if transpose and block[0] == 1 else (None, 0, 0, 0)
        _check(lib.b200_fp8_quantize(in_type, ct, block[0], m, k, groups, x.data_ptr(), ld(x), e(x), q.data_ptr(),
                                     ld(q), e(q), s.data_ptr(), *s.stride()[-2:], e(s), *t_args, *st_args,
                                     _stream_ptr(stream)))
    return (q, s, qt, st) if transpose else (q, s)


def gemm_f32(A, B, out=None, mode=F32_AUTO, stream=None, accumulate=False):
    """C = A*B, or C += A*B into `out` when accumulate is set (b200_gemm_f32_acc)."""
    import torch
    assert A.dtype == torch.float32 and B.dtype == torch.float32 and A.is_cuda and B.is_cuda
    m, k = A.shape
    k2, n = B.shape
    assert k == k2
    if out is None:
        out = torch.empty((m, n), dtype=torch.float32, device=A.device)
    fn = lib.b200_gemm_f32_acc if accumulate else lib.b200_gemm_f32
    assert not accumulate or out is not None
    _check(fn(m, n, k, A.data_ptr(), _ld(A), B.data_ptr(), _ld(B), out.data_ptr(), _ld(out), mode, _stream_ptr(stream)))
    return out


def gemm_f32_ex(alpha, A, B, beta, out, mode=F32_AUTO, stream=None):
    """out = alpha * A*B + beta * out (b200_gemm_f32_ex; cuBLAS sgemm semantics, cuda/MMult_cuBLAS_1.cpp:11-19)."""
    m, k = A.shape
    n = B.shape[1]
    _check(lib.b200_gemm_f32_ex(m, n, k, alpha, A.data_ptr(), _ld(A), B.data_ptr(), _ld(B), beta, out.data_ptr(), _ld(out),
                                mode, _stream_ptr(stream)))
    return out


def mxf4_quantize(X, transpose=False, stream=None):
    """fp32 CUDA matrix -> (q, sf, rows, k): packed E2M1 rows + UE8M0 scale atoms (b200_mxf4_quantize_a / _b).
    transpose=False: X is A (m x k), rows = m.  transpose=True: X is B (k x n) and the result is B^T (rows = n)."""
    import torch
    assert X.dtype == torch.float32 and X.is_cuda and X.dim() == 2
    r, c = X.shape
    rows, k = (c, r) if transpose else (r, c)
    q = torch.empty(lib.b200_mxf4_q_bytes(rows, k), dtype=torch.uint8, device=X.device)
    sf = torch.empty(lib.b200_mxf4_sf_bytes(rows, k), dtype=torch.uint8, device=X.device)
    fn = lib.b200_mxf4_quantize_b if transpose else lib.b200_mxf4_quantize_a
    _check(fn(r, c, X.data_ptr(), _ld(X), q.data_ptr(), sf.data_ptr(), _stream_ptr(stream)))
    return q, sf, rows, k


def gemm_mxf4(qa, sfa, qb, sfb, m, n, k, out=None, stream=None):
    """C (m x n fp32) = dequant(A_q) * dequant(B_q)^T from mxf4_quantize outputs (b200_gemm_mxf4)."""
    import torch
    if out is None:
        out = torch.empty((m, n), dtype=torch.float32, device=qa.device)
    _check(lib.b200_gemm_mxf4(m, n, k, qa.data_ptr(), sfa.data_ptr(), qb.data_ptr(), sfb.data_ptr(), out.data_ptr(), _ld(out),
                              _stream_ptr(stream)))
    return out


def gemm_bf16(A, B, out=None, out_dtype=None, stream=None):
    import torch
    assert A.dtype == torch.bfloat16 and B.dtype == torch.bfloat16 and A.is_cuda and B.is_cuda
    m, k = A.shape
    k2, n = B.shape
    assert k == k2
    if out is None:
        out = torch.empty((m, n), dtype=out_dtype or torch.float32, device=A.device)
    ot = OUT_F32 if out.dtype == torch.float32 else OUT_BF16
    assert out.dtype in (torch.float32, torch.bfloat16)
    _check(lib.b200_gemm_bf16(m, n, k, A.data_ptr(), _ld(A), B.data_ptr(), _ld(B), out.data_ptr(), _ld(out),
                              ot, _stream_ptr(stream)))
    return out


class PackedB:
    """Pre-split B (b200_gemm_f32_pack_b): holds the handle, frees it with the object."""

    def __init__(self, B, mode=F32_AUTO, stream=None):
        import torch
        assert B.dtype == torch.float32 and B.is_cuda and B.dim() == 2
        self.k, self.n = B.shape
        self.handle = _vp()
        _check(lib.b200_gemm_f32_pack_b(self.k, self.n, B.data_ptr(), _ld(B), mode, C.byref(self.handle),
                                        _stream_ptr(stream)))

    def close(self):
        if getattr(self, "handle", None):
            lib.b200_gemm_f32_pack_free(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:      # interpreter shutdown: module globals may already be gone
            pass


class PackedA:
    """Pre-split A (b200_gemm_f32_pack_a, F16X2): holds the handle, frees it with the object."""

    def __init__(self, A, mode=F32_AUTO, stream=None):
        import torch
        assert A.dtype == torch.float32 and A.is_cuda and A.dim() == 2
        self.m, self.k = A.shape
        self.handle = _vp()
        _check(lib.b200_gemm_f32_pack_a(self.m, self.k, A.data_ptr(), _ld(A), mode, C.byref(self.handle),
                                        _stream_ptr(stream)))

    def close(self):
        if getattr(self, "handle", None):
            lib.b200_gemm_f32_pack_free_a(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def gemm_f32_packed_ab(packedA, packedB, out, a_k0=0, stream=None, accumulate=False):
    """C (+)= A[:, a_k0:a_k0+k] * B from two pre-split operands (b200_gemm_f32_packed_ab)."""
    _check(lib.b200_gemm_f32_packed_ab(packedA.m, packedB.n, packedB.k, packedA.handle, a_k0, packedB.handle,
                                       out.data_ptr(), _ld(out), 1 if accumulate else 0, _stream_ptr(stream)))
    return out


def gemm_f32_packed(A, packedB, out=None, stream=None, accumulate=False):
    import torch
    assert A.dtype == torch.float32 and A.is_cuda
    m, k = A.shape
    if out is None:
        assert not accumulate
        out = torch.empty((m, packedB.n), dtype=torch.float32, device=A.device)
    _check(lib.b200_gemm_f32_packed(m, packedB.n, k, A.data_ptr(), _ld(A), packedB.handle, out.data_ptr(), _ld(out),
                                    1 if accumulate else 0, _stream_ptr(stream)))
    return out


def gemm_s8s8_requant(A, B, scales, bias=None, out=None, stream=None):
    """int8 x int8 -> int8 with per-row scales / bias (aarch64-int8/int8kernel_m4.S:40,386-426)."""
    import torch
    assert A.dtype == torch.int8 and B.dtype == torch.int8 and A.is_cuda and B.is_cuda
    m, k = A.shape
    k2, n = B.shape
    assert k == k2
    assert scales.dtype == torch.float32 and scales.is_cuda and scales.is_contiguous() and scales.numel() == m
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_cuda and bias.is_contiguous() and bias.numel() == m
    if out is None:
        out = torch.empty((m, n), dtype=torch.int8, device=A.device)
    assert out.dtype == torch.int8
    _check(lib.b200_gemm_s8s8_requant(m, n, k, A.data_ptr(), _ld(A), B.data_ptr(), _ld(B), out.data_ptr(), _ld(out),
                                      scales.data_ptr(), bias.data_ptr() if bias is not None else None,
                                      _stream_ptr(stream)))
    return out


def gemm_s8s32(A, B, out=None, stream=None):
    import torch
    assert A.dtype == torch.int8 and B.dtype == torch.int8 and A.is_cuda and B.is_cuda
    m, k = A.shape
    k2, n = B.shape
    assert k == k2
    if out is None:
        out = torch.empty((m, n), dtype=torch.int32, device=A.device)
    _check(lib.b200_gemm_s8s32(m, n, k, A.data_ptr(), _ld(A), B.data_ptr(), _ld(B), out.data_ptr(), _ld(out),
                               _stream_ptr(stream)))
    return out


def convert_f32_to_bf16(src, stream=None):
    import torch
    out = torch.empty(src.shape, dtype=torch.bfloat16, device=src.device)
    _check(lib.b200_convert_f32_to_bf16(src.data_ptr(), out.data_ptr(), src.numel(), _stream_ptr(stream)))
    return out
