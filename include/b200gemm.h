/*
 * b200gemm.h — C ABI of the H100-native (sm_90a) row-major GEMM (libb200gemm.so).
 *
 * This header is the drop-in boundary for the hot path of
 * tpoisonooo/how-to-optimize-gemm: the free function MY_MMult that the
 * reference's harness links against exactly one object for.  Every entry point
 * below cites the reference interface it stands behind:
 *
 *   b200_gemm_f32     <- cuda/test_MMult.cpp:13-14  (10-arg MY_MMult, device
 *                        pointers, C = A*B; wrapper cuda/MMult_cuda_12.cu:228-235)
 *   b200_gemm_f32_host<- aarch64/MMult0.cpp:3-23 / aarch64/test_MMult.cpp:17
 *                        (9-arg MY_MMult, host pointers, C += A*B)
 *   b200_gemm_bf16    <- same contraction, bf16 operands (BASELINE config 3; no
 *                        reference precedent, semantics of cuda/test_MMult.cpp)
 *   b200_gemm_s8s32   <- aarch64-int8/MMult_4x8_21.c:81-86 (12-arg MY_MMult,
 *                        int8 x int8 -> int32, C = A*B, any m,n,k)
 *   b200_gemm_s8s32_host <- aarch64-int8/test_MMult.c:9,98 (host pointers)
 *   b200_gemm_s8s8_requant <- aarch64-int8/int8kernel_m4.S:40 (int8kernel_m4_requant:
 *                        int8 x int8 -> int8 through per-row scales / bias, :386-426)
 *
 * All matrices are ROW-MAJOR: A is m x k (leading dimension lda >= k),
 * B is k x n (ldb >= n), C is m x n (ldc >= n); leading dimensions are in
 * ELEMENTS.  The reference only ever passes lda=k, ldb=n, ldc=n
 * (cuda/test_MMult.cpp:62) and silently ignores them
 * (cuda/MMult_cuda_12.cu:231-234); this library honours them.
 *
 * Device entry points are fully asynchronous on `stream` (a cudaStream_t passed
 * as void*; NULL = the legacy default stream the reference harness uses,
 * cuda/test_MMult.cpp:98-110), never synchronise or allocate in steady state (see
 * b200_gemm_reserve_workspace for the first call) and may be called on any stream of any
 * sm_90 device (per-device state; make the device current on the calling thread; a thread needs no CUDA call of
 * its own before the first: that call makes the device's primary context current).  They return 0 on success or a cudaError_t /
 * negative B200_ERR_* code.  There is NO CPU fallback: without a CUDA device of
 * compute capability 9.x every compute entry point returns
 * B200_ERR_NO_DEVICE.
 */
#ifndef B200GEMM_H_
#define B200GEMM_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes (negative; positive values are cudaError_t) ------------ */
#define B200_OK                 0
#define B200_ERR_BAD_ARG       -1   /* null pointer, negative size, ld too small */
#define B200_ERR_NO_DEVICE     -2   /* no sm_90 device / driver entry point missing */
#define B200_ERR_UNSUPPORTED   -3   /* mode not available for this dtype */
#define B200_ERR_TENSORMAP     -4   /* cuTensorMapEncodeTiled rejected the operand */
#define B200_ERR_NCCL          -5   /* libnccl missing or an NCCL call failed: b200_nccl_last_error() */

/* ---- fp32 precision modes (the SURVEY §7 H1 decision, made explicit) ------ */
enum b200_f32_mode {
  B200_F32_STRICT = 0,   /* CUDA-core FFMA, fp32 multiply-add, k ascending: the
                            arithmetic of cuda/MMult_cuda_12.cu:200-206          */
  B200_F32_TF32   = 1,   /* one tf32 wgmma pass (10-bit mantissa inputs, fp32
                            accumulate)                                           */
  B200_F32_BF16X3 = 2,   /* split-bf16: a=a1+a2+a3, 6 bf16 wgmma products per
                            k-step, two-level accumulation (K chunks of 512, each a
                            fresh accumulator added with a rounded fp32 add to a
                            running sum held in registers): fp32-class error on the
                            tensor cores, elementwise.  The round-1 default.      */
  B200_F32_BF16X2 = 3,   /* split-bf16: a=a1+a2, 3 products, ~2^-17 relative       */
  B200_F32_AUTO   = 4,   /* library default: F16X2 unless the environment variable
                            B200GEMM_F32_MODE or b200_gemm_set_default_f32_mode
                            says otherwise; problems up to ~512^3 with TMA-able
                            operands take the single-launch STRICT kernel, problems
                            up to ~1100^3 the two-launch BF16X3 path               */
  B200_F32_F16X2  = 5    /* scaled split-fp16: rows of A / columns of B are scaled by
                            exact powers of two into [-1,1], a'=h1+h2 in fp16 (22
                            bits), 3 fp16 wgmma products, two-level
                            accumulation, epilogue unscales.  fp32-class NORMWISE
                            error (elements far below their row/column maximum keep
                            absolute, not relative, precision): half the tensor-core
                            work of BF16X3 at the same measured error.
                            THE LIBRARY DEFAULT.                                   */
};
/* Range contract of the fp32 modes (tests/test_fp32_range_gpu.py), over the whole fp32
 * range including subnormals, FLT_MAX, inf and NaN:
 *  - C(i,j) is non-finite exactly where the IEEE result is: an inf or NaN in row i of A or
 *    column j of B, or a result beyond FLT_MAX.  No other element is contaminated.  The split
 *    modes may return NaN where IEEE gives +-inf: they form inf*(b1 + b2) as inf*b1 + inf*b2.
 *  - Finite results: STRICT is one fused multiply-add chain per element (bit-exact against the
 *    naive reference); BF16X3 within 2^-22 (|A||B|)ij, BF16X2 within 2^-14 (|A||B|)ij, TF32
 *    within 2^-9 (|A||B|)ij, elementwise; F16X2 within 2^-20 K max|A(i,:)| max|B(:,j)|
 *    (normwise per row and column, subnormal and near-FLT_MAX maxima included); each plus
 *    its fp32 accumulation error.  In the bf16 and tf32 modes an operand below about 2^-110
 *    loses bits absolutely (its lower planes fall under the bf16 subnormal quantum 2^-133):
 *    add 2^-133 (sum_k |A(i,k)| + sum_k |B(k,j)|).
 *  - The H100 tensor cores keep subnormal bf16, tf32 and fp16 inputs and subnormal fp32
 *    products and sums (observed on an H100 80GB HBM3): nothing is flushed to zero.        */

/* ---- output selector of the 16-bit GEMMs ----------------------------------- */
enum b200_out_type {
  B200_OUT_F32  = 0,     /* C written as float   (4 B/elem): bf16 and fp16 operands */
  B200_OUT_BF16 = 1,     /* C written as bf16    (2 B/elem): bf16 operands only     */
  B200_OUT_F16  = 2      /* C written as fp16    (2 B/elem): fp16 operands only     */
};

/* Library / device ---------------------------------------------------------- */
const char* b200_gemm_version(void);
/* 0 if a usable sm_90 device is current, else B200_ERR_NO_DEVICE. */
int  b200_gemm_device_ok(void);
/* Human-readable text for a code returned by this library. */
const char* b200_gemm_strerror(int code);
/* Name of the kernel the last call on this thread dispatched to
 * ("tc_bf16_128x256", "ffma_128x128", ...), for tests and bench evidence. */
const char* b200_gemm_last_kernel(void);
/* Number of kernel launches this library has issued since load. */
unsigned long long b200_gemm_launch_count(void);
int  b200_gemm_default_f32_mode(void);
void b200_gemm_set_default_f32_mode(int mode);

/* The split-precision fp32 modes keep the planes of A and B in a per-device, grow-only workspace.  Its first
 * use and every growth allocate (and synchronise the device); steady-state calls never do.  Reserve it up front
 * — b200_gemm_reserve_workspace(b200_gemm_workspace_bytes(m, n, k, mode)) on the device that will run the
 * calls — to keep even the first call allocation-free (e.g. ahead of CUDA-graph capture).
 * b200_gemm_workspace_bytes(m, n, k, mode) is b200_gemm_workspace_bytes_op(B200_OP_N, B200_OP_N, m, n, k, mode):
 * for an explicit mode exactly what its route reserves, for AUTO the largest of the routes AUTO may take at this
 * size (plain or with a general alpha / beta).  State is per device:
 * one process may drive several GPUs (make the device current on the calling thread).  Calls on different
 * streams (or host threads) of one device are ordered by events, not by the host, on what they share: the
 * workspace, the F16X2 column maxima and the K-split flag slots.  Under stream capture the flag slots are not
 * ordered: a replayed graph must not run beside split-tail calls on other streams of the device.
 * The same workspace holds B^T for B200_F32_TF32 (counted by b200_gemm_workspace_bytes) and for the int8 entry
 * points (n * k16 bytes, k16 = k rounded up to 16), and the bf16 expansions of both operands for b200_gemm_mxf4
 * (round1024(2 * m * kpad) + 2 * kpad * n8 bytes, kpad = k rounded up to 128, n8 = n rounded up to 8): reserve
 * that much before the first such call to keep it allocation-free too. */
size_t b200_gemm_workspace_bytes(int m, int n, int k, int precision_mode);
int    b200_gemm_reserve_workspace(size_t bytes);

/* fp32: C = A*B.  Replaces MY_MMult(cublasHandle_t,m,n,k,dA,lda,dB,ldb,dC,ldc)
 * (cuda/test_MMult.cpp:13-14,100-103).  DEVICE pointers. */
int b200_gemm_f32(int m, int n, int k,
                  const float* dA, int lda, const float* dB, int ldb,
                  float* dC, int ldc, int precision_mode, void* stream);

/* fp32: C += A*B on DEVICE pointers — the CPU harnesses' contract (aarch64/MMult0.cpp:16) without
 * the staging copies; also what lets a K-sliced operand stream (B arriving in row chunks over
 * NVLink) be consumed chunk by chunk.  STRICT keeps one fused chain per element starting from C(i,j);
 * the tensor-core modes fold their fp32 partial sums into C with rounded adds. */
int b200_gemm_f32_acc(int m, int n, int k,
                      const float* dA, int lda, const float* dB, int ldb,
                      float* dC, int ldc, int precision_mode, void* stream);

/* fp32: C = alpha * A*B + beta * C on DEVICE pointers — the contract of the reference's cuBLAS comparator
 * (cublasSgemm, cuda/MMult_cuBLAS_1.cpp:11-19; the harness only ever passes alpha = 1, beta = 0).  beta == 0
 * never reads C; alpha == 0 never reads A or B (one element-wise pass C = beta * C).  (1, 0) and (1, 1) are
 * b200_gemm_f32 / b200_gemm_f32_acc exactly; any other pair is fused into the epilogue of every kernel
 * (tensor-core, strict FFMA and generic): the product is accumulated from zero and stored as
 * fma(beta, C, alpha * AB), so no intermediate such as beta / alpha can overflow. */
int b200_gemm_f32_ex(int m, int n, int k, float alpha,
                     const float* dA, int lda, const float* dB, int ldb, float beta,
                     float* dC, int ldc, int precision_mode, void* stream);

/* 16-bit operands: C = alpha * op(A)*op(B) + beta * C on DEVICE pointers — cublasGemmEx's contract for bf16 and fp16
 * (cuda/MMult_cuBLAS_2.cpp).  op_a / op_b and the leading dimensions are those of b200_gemm_f32_op (below).
 *   b200_gemm_bf16_ex: bf16 operands, out_type B200_OUT_F32 or B200_OUT_BF16.
 *   b200_gemm_f16_ex:  IEEE fp16 operands, out_type B200_OUT_F32 or B200_OUT_F16.
 * Errors: an out_type that does not fit the operand type (F16 for bf16, BF16 for fp16, anything else), an op other
 * than 0 or 1, an ld below its op's minimum or a null pointer is B200_ERR_BAD_ARG; m == 0 or n == 0 is a no-op.
 * (alpha, beta) = (1, 0) is b200_gemm_bf16_op / b200_gemm_f16 exactly: same kernel, kernel name, launches and bits.
 * Any other pair is fused into the epilogue of the tensor-core and the generic kernel: the fp32 accumulator x is
 * stored as round_out(fma(beta, float(C), alpha * x)).  float(C) is exact for 16-bit C; round_out is the identity
 * for fp32 C and one round-to-nearest-even to bf16 / fp16 otherwise.  beta == 0 never reads C (a NaN already in C
 * stays out of the result); alpha == 0 or k == 0 never reads A or B: one element-wise pass C = round_out(beta *
 * float(C)), zeros when beta == 0.  fp16 C rounds to nearest even and overflows to +-inf, as torch's .half() does.
 * fp32 C may take the K-split tail (beta * C is folded by the first K part only); 16-bit C never does, and neither does
 * a call with a bias or an activation (b200_gemm_bf16_epi / _f16_epi, below).  No workspace.
 * Kernels: "tc_f16_128x{256,192,128}" (fp32 C) and "tc_f16_of16_128x..." (fp16 C), with the layout infix _nt / _tn
 * / _tt as for bf16; operands that TMA cannot read take "generic_f16_64x64" (CUDA cores, sequential k). */
int b200_gemm_bf16_ex(int op_a, int op_b, int m, int n, int k, float alpha,
                      const uint16_t* dA, int lda, const uint16_t* dB, int ldb, float beta,
                      void* dC, int ldc, int out_type, void* stream);
int b200_gemm_f16_ex(int op_a, int op_b, int m, int n, int k, float alpha,
                     const uint16_t* dA, int lda, const uint16_t* dB, int ldb, float beta,
                     void* dC, int ldc, int out_type, void* stream);

/* Strided-batched 16-bit GEMM (cublasGemmStridedBatchedEx; torch.bmm / torch.baddbmm): for b = 0 .. batch - 1,
 *   C_b = round_out(fma(beta, float(C_b), alpha * op(A_b) * op(B_b))),   X_b = X + b * stride_x  (strides in elements).
 * Each entry follows the rules of b200_gemm_bf16_ex / b200_gemm_f16_ex exactly: ops, minimum ld, out_type pairing,
 * beta == 0 never reads C, alpha == 0 or k == 0 never reads A or B.  Further rules, each checked before the device is
 * touched:
 *   - batch < 0 or a negative stride is B200_ERR_BAD_ARG; batch == 0, m == 0 or n == 0 is a no-op, NULL pointers
 *     included; a NULL pointer with work to do is B200_ERR_BAD_ARG.
 *   - stride_a and stride_b may be 0: one operand broadcast over the batch.  They may also be smaller than an entry of
 *     the operand (overlapping input entries); such a call runs on the generic kernel.
 *   - batch > 1 with stride_c < (m - 1) * ldc + n is B200_ERR_BAD_ARG: two entries of C would overlap.
 *   - batch * ceil(m / 128) * ceil(n / 128) * 4 above 2^31 - 1 is B200_ERR_BAD_ARG: the kernel counts the batch's
 *     tiles (and their K-split parts) in an int.  So is (batch - 1) * stride above 2^60 elements for any operand.
 *   - batch == 1 is the _ex call exactly: same kernel, kernel name, launches and bits.
 * Every other call is one launch for the whole batch (see the launch table below):
 *   - 16-byte-aligned bases with lda, ldb, stride_a and stride_b multiples of 16 bytes, each input stride 0 or at least
 *     its entry's rows x ld as stored: the persistent tensor-core kernel walks the tiles of every entry, entry outermost,
 *     tile width chosen for the whole batch's tile count.  fp32 C may take the K-split tail on the last partial round
 *     of the whole batch; 16-bit C never does.  Kernels "tc_bf16_bat_128x256", "tc_bf16_obf16_bat_nt_128x192",
 *     "tc_f16_bat_tn_128x128", "tc_f16_of16_bat_tt_128x256", ...
 *   - any other operands: the generic kernel, "generic_bf16_bat_64x64" / "generic_f16_bat_64x64", every entry bit for
 *     bit as the 2-D generic kernel computes it.
 *   - alpha == 0 or k == 0: one element-wise pass over every entry, "fill_zero_bat" (beta == 0) or "scale_inplace_bat".
 * No workspace.  Operand types and out_type as for _bf16_ex / _f16_ex. */
int b200_gemm_bf16_batched(int op_a, int op_b, int m, int n, int k, float alpha,
                           const uint16_t* dA, int lda, long long stride_a,
                           const uint16_t* dB, int ldb, long long stride_b, float beta,
                           void* dC, int ldc, long long stride_c, int batch, int out_type, void* stream);
int b200_gemm_f16_batched(int op_a, int op_b, int m, int n, int k, float alpha,
                          const uint16_t* dA, int lda, long long stride_a,
                          const uint16_t* dB, int ldb, long long stride_b, float beta,
                          void* dC, int ldc, long long stride_c, int batch, int out_type, void* stream);

/* Grouped 16-bit GEMM (torch._grouped_mm(x, W, offs=offs); a mixture-of-experts layer): the rows routed to each group
 * are stacked in one row-major A (total_m x k, lda >= k), the groups' B_g lie at dB + g * stride_b (elements), and
 * dOffs holds `groups` int32 cumulative end rows on the DEVICE.  With end_{-1} = 0 and
 *   end_g = min(max(dOffs[g], end_{g-1}), total_m),
 * rows [end_{g-1}, end_g) of C (total_m x n, row-major, ldc >= n) become
 *   round_out(fma(beta, float(C), alpha * A_rows * op(B_g))).
 * op_b follows _ex: B200_OP_N, each B_g is k x n (ldb >= n); B200_OP_T, each B_g is stored n x k (ldb >= k), which is
 * how a (groups, n, k) weight W is passed for x @ W_g^T.  A is always N.
 * dOffs is read only on the device, after the work the stream already holds (a routing kernel may write it): the host
 * never reads it and never synchronises, so the call can be captured in a CUDA graph and replayed with new offsets.
 * The clamp makes every offset legal: non-monotone, negative or too-large offsets give the groups above (an empty
 * group where an offset goes back), and no row outside [0, total_m) is ever read or written.  Rows at or after
 * end_{groups-1} are never written.  Each group is bit for bit the _ex call on a contiguous copy of its rows of A and
 * on B_g, at the same tile width (the tensor-core kernel never takes the K-split tail, so the _ex call with it off).
 * Argument rules, each checked before the device is touched:
 *   - the _ex rules for an m = total_m call with op_a = N: op_b, minimum ld, out_type pairing; beta == 0 never reads C;
 *     alpha == 0 or k == 0 never reads A or B.
 *   - negative sizes, groups or stride_b, and groups > 1024, are B200_ERR_BAD_ARG.
 *   - groups > 1 with stride_b < (rows of B_g as stored) * ldb is B200_ERR_BAD_ARG: the B_g may not overlap or be
 *     broadcast.  (groups == 1 ignores stride_b.)  So is (groups - 1) * stride_b above 2^60 elements.
 *   - (ceil(total_m / 128) + groups) * ceil(n / 128) above 2^30 - 1 is B200_ERR_BAD_ARG: the kernel counts its tile
 *     bound in an int.
 *   - groups == 0, total_m == 0 or n == 0 is a no-op, NULL pointers included; a NULL pointer with work to do, dOffs
 *     included, is B200_ERR_BAD_ARG.
 * Routes, each one launch, no workspace:
 *   - 16-byte-aligned A and B with lda, ldb and stride_b multiples of 16 bytes: the persistent tensor-core kernel.  It
 *     builds its tile schedule from dOffs on the device; the host sizes its grid and tile width for the bound
 *     ceil(total_m / 128) + groups tile rows (each group adds at most one partial tile), which
 *     b200_gemm_debug_last_schedule reports as tiles (a bound, not the tiles the offsets give), with split 1.  Kernels
 *     "tc_bf16_grp_128x256", "tc_bf16_obf16_grp_nt_128x192", "tc_f16_grp_128x128", "tc_f16_of16_grp_nt_128x256", ...
 *   - any other operands: the generic kernel, "generic_bf16_grp_64x64" / "generic_f16_grp_64x64", every group bit for
 *     bit as the 2-D generic kernel computes its rows.
 *   - alpha == 0 or k == 0: one element-wise pass over rows [0, end_{groups-1}), "fill_zero_grp" (beta == 0) or
 *     "scale_inplace_grp".
 * No bias or activation epilogue. */
int b200_gemm_bf16_grouped(int op_b, int total_m, int n, int k, float alpha,
                           const uint16_t* dA, int lda,
                           const uint16_t* dB, int ldb, long long stride_b,
                           const int32_t* dOffs, int groups, float beta,
                           void* dC, int ldc, int out_type, void* stream);
int b200_gemm_f16_grouped(int op_b, int total_m, int n, int k, float alpha,
                          const uint16_t* dA, int lda,
                          const uint16_t* dB, int ldb, long long stride_b,
                          const int32_t* dOffs, int groups, float beta,
                          void* dC, int ldc, int out_type, void* stream);

/* K-grouped 16-bit GEMM (torch._grouped_mm(dy.t(), x, offs=offs), 2-D x 2-D; the weight gradient dW_g = dy_g^T x_g of
 * a mixture-of-experts layer): the offsets split the contraction dimension, and every group writes a whole C_g.
 * op(A) is m x total_k and op(B) is total_k x n, each stored as for _ex: op_a = B200_OP_T, A stored total_k x m
 * (lda >= m, the dy.t() of a row-major dy); op_b = B200_OP_N, B is total_k x n (ldb >= n, a row-major x); N and T
 * otherwise as in b200_gemm_f32_op.  dOffs holds `groups` int32 cumulative ends on the DEVICE; with end_{-1} = 0,
 *   end_g = min(max(dOffs[g], end_{g-1}), total_k),   k_g = end_g - end_{g-1},
 *   C_g = round_out(fma(beta, float(C_g), alpha * op(A)[:, end_{g-1}:end_g] * op(B)[end_{g-1}:end_g, :]))
 * for every g < groups, with C_g (m x n, row-major, ldc >= n) at dC + g * stride_c (elements).  Every group is
 * written: an empty one (k_g = 0) stores exactly what _ex with k == 0 stores, raw +0 when beta == 0 (C unread) and
 * round_out(beta * float(C)) otherwise.  Each C_g is bit for bit the _ex call with k = k_g on contiguous copies of its
 * K range of A and B, at the same tile width (the _ex call with the K-split tail off).  The host never reads dOffs and
 * never synchronises, so the call can be captured in a CUDA graph and replayed with new offsets.
 * Argument rules, each checked before the device is touched:
 *   - the _ex rules for an (m, n, total_k) call: ops, minimum ld, out_type pairing; beta == 0 never reads C; alpha == 0
 *     or total_k == 0 never reads A or B.
 *   - negative sizes, groups or stride_c, groups > 1024, and total_k > 2^31 - 65 (K row coordinates up to end + 64
 *     stay within int32) are B200_ERR_BAD_ARG.
 *   - groups > 1 with stride_c < (m - 1) * ldc + n is B200_ERR_BAD_ARG: two C_g would overlap.  So is
 *     (groups - 1) * stride_c above 2^60 elements.
 *   - groups * ceil(m / 128) * ceil(n / 128) above 2^30 - 1 is B200_ERR_BAD_ARG: the kernel counts its tiles in an int.
 *   - groups == 0, m == 0 or n == 0 is a no-op, NULL pointers included; a NULL pointer with work to do, dOffs
 *     included, is B200_ERR_BAD_ARG.  total_k == 0 is not a no-op: every C_g becomes beta * C_g, or zeros.
 * Routes, each one launch, no workspace, no K-split tail:
 *   - (op_a, op_b) = (T, N) with 16-byte-aligned A and B and lda, ldb multiples of 16 bytes: the persistent tensor-core
 *     kernel over every group's tiles, group outermost, tile width chosen for groups x m x n as for a batch;
 *     b200_gemm_debug_last_schedule reports tiles = groups * ceil(m / 128) * ceil(n / BN), split 1.  Kernels
 *     "tc_bf16_kgrp_tn_128x256", "tc_bf16_obf16_kgrp_tn_128x192", "tc_f16_kgrp_tn_128x128",
 *     "tc_f16_of16_kgrp_tn_128x256", ...
 *   - every other layout, and operands TMA cannot read: the generic kernel, "generic_bf16_kgrp_64x64" /
 *     "generic_f16_kgrp_64x64", every group bit for bit as the 2-D generic kernel computes it.
 *   - alpha == 0 or total_k == 0: one element-wise pass over every C_g, "fill_zero_bat" (beta == 0) or
 *     "scale_inplace_bat".
 * No bias or activation epilogue. */
int b200_gemm_bf16_grouped_k(int op_a, int op_b, int m, int n, int total_k, float alpha,
                             const uint16_t* dA, int lda, const uint16_t* dB, int ldb,
                             const int32_t* dOffs, int groups, float beta,
                             void* dC, int ldc, long long stride_c, int out_type, void* stream);
int b200_gemm_f16_grouped_k(int op_a, int op_b, int m, int n, int total_k, float alpha,
                            const uint16_t* dA, int lda, const uint16_t* dB, int ldb,
                            const int32_t* dOffs, int groups, float beta,
                            void* dC, int ldc, long long stride_c, int out_type, void* stream);

/* 16-bit operands with a bias vector and an activation fused into the epilogue (cuBLASLt's CUBLASLT_EPILOGUE_BIAS,
 * _RELU_BIAS, _GELU_BIAS): C = round_out(act(alpha * op(A)*op(B) + beta * C + bias)), what a PyTorch
 * act(F.linear(x, W, b)) computes, in one launch.  Arguments as b200_gemm_bf16_ex / b200_gemm_f16_ex, plus:
 *   dBias: n contiguous elements of the operand type (bf16 bits for _bf16_epi, fp16 bits for _f16_epi), one per column
 *          of C, at any 2-byte-aligned device address; NULL = no bias.
 *   act:   one of the B200_ACT_* codes below; any other value is B200_ERR_BAD_ARG.
 * Per element, in fp32, with x the fp32 accumulator:
 *   1. t = fma(beta, float(C), alpha * x), the _ex rule (beta == 0 never reads C);
 *   2. t = t + float(bias[j]), one round-to-nearest add, skipped when dBias is NULL;
 *   3. y = act(t);
 *   4. C = round_out(y): the identity for fp32 C, one round-to-nearest-even to bf16 / fp16 otherwise (fp16 overflows
 *      to +-inf).
 * B200_ACT_RELU is t < 0 ? +0 : t (NaN stays NaN, -0 stays -0, as torch.relu).  The two GELUs are evaluated in fp32
 * with CUDA's erfcf / tanhf (GELU as 0.5 t erfc(-t / sqrt 2), which keeps relative accuracy for negative t); at the
 * ends of the range they give the limits of the function: +inf -> +inf, -inf -> -0, NaN -> NaN (torch on the CPU
 * returns NaN for gelu(+-inf)).  The tensor-core and the generic kernel share one activation function, so both routes
 * give the same bits for the same t.
 * dBias == NULL with B200_ACT_NONE is the _ex call exactly: same kernel, kernel name, launches and bits.  The other
 * argument rules of _ex apply (out_type pairing, ops, minimum ld, null pointers); m == 0 or n == 0 is a no-op, a NULL
 * bias included.  alpha == 0 or k == 0 never reads A or B: one element-wise pass stores round_out(act(beta * float(C) +
 * bias[j])), where beta == 0 contributes +0 and does not read C (so the result is act(+0 + bias[j]) down every row).
 * A call with a bias or an activation never takes the K-split tail, fp32 C included: the activation is not linear and
 * must see the complete sum.  Every layout is one launch on the tensor cores, tile widths 256 / 192 / 128 as for _ex;
 * kernels are named with "_epi" after the C-type part ("tc_bf16_epi_128x256", "tc_bf16_obf16_epi_nt_128x192",
 * "tc_f16_epi_tn_128x128", "tc_f16_of16_epi_tt_128x256").  Operands that TMA cannot read take the generic kernel
 * ("generic_bf16_64x64" / "generic_f16_64x64", one launch).  No workspace. */
#define B200_ACT_NONE      0   /* bias only (or nothing: then this is the _ex call)                                 */
#define B200_ACT_RELU      1
#define B200_ACT_GELU      2   /* x * Phi(x), the erf form (torch's default nn.GELU)                                */
#define B200_ACT_GELU_TANH 3   /* 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))): cuBLASLt's GELU, torch's
                                  approximate='tanh'                                                                 */
int b200_gemm_bf16_epi(int op_a, int op_b, int m, int n, int k, float alpha,
                       const uint16_t* dA, int lda, const uint16_t* dB, int ldb, float beta,
                       void* dC, int ldc, int out_type, const uint16_t* dBias, int act, void* stream);
int b200_gemm_f16_epi(int op_a, int op_b, int m, int n, int k, float alpha,
                      const uint16_t* dA, int lda, const uint16_t* dB, int ldb, float beta,
                      void* dC, int ldc, int out_type, const uint16_t* dBias, int act, void* stream);

/* fp32 with HOST pointers and the CPU harness contract C += A*B
 * (aarch64/MMult0.cpp:11-19; harness zeroes C first, aarch64/test_MMult.cpp:107).
 * Stages H2D, runs b200_gemm_f32 on the device, adds into C on the device,
 * copies back, synchronises.  Plumbing/parity only, never a reported number. */
int b200_gemm_f32_host(int m, int n, int k,
                       const float* A, int lda, const float* B, int ldb,
                       float* C, int ldc, int precision_mode);

/* bf16 operands (raw uint16 bit patterns), fp32 accumulate; C is float or bf16
 * according to out_type.  DEVICE pointers. */
int b200_gemm_bf16(int m, int n, int k,
                   const uint16_t* dA, int lda, const uint16_t* dB, int ldb,
                   void* dC, int ldc, int out_type, void* stream);

/* IEEE fp16 operands (raw uint16 bit patterns), fp32 accumulate; C is float (B200_OUT_F32) or fp16 (B200_OUT_F16,
 * round to nearest even, overflow to +-inf).  The fp16 twin of b200_gemm_bf16: same tiles, schedule and routes.
 * DEVICE pointers. */
int b200_gemm_f16(int m, int n, int k,
                  const uint16_t* dA, int lda, const uint16_t* dB, int ldb,
                  void* dC, int ldc, int out_type, void* stream);

/* int8 x int8 -> int32, exact: C = A*B (aarch64-int8/README.md:8; oracle
 * aarch64-int8/REF_MMult.c:10-23).  DEVICE pointers. */
int b200_gemm_s8s32(int m, int n, int k,
                    const int8_t* dA, int lda, const int8_t* dB, int ldb,
                    int32_t* dC, int ldc, void* stream);

/* int8 with HOST pointers: what aarch64-int8/test_MMult.c:98 passes. */
int b200_gemm_s8s32_host(int m, int n, int k,
                         const int8_t* A, int lda, const int8_t* B, int ldb,
                         int32_t* C, int ldc);

/* ---- transposed operands (cuBLAS transa / transb; chgemm's trans / trans_w, aarch64-int8/MMult_4x8_21.c:45-71) ----
 * C = alpha * op(A) * op(B) + beta * C, C row-major m x n (ldc >= n), each operand stored row-major either as is or
 * transposed:
 *   op_a = B200_OP_N: A is m x k, lda >= k;   B200_OP_T: A is stored as A^T, k x m, lda >= m
 *   op_b = B200_OP_N: B is k x n, ldb >= n;   B200_OP_T: B is stored as B^T, n x k, ldb >= k
 * (a PyTorch caller's x @ W.t() with W of shape n x k is op_b = B200_OP_T, ldb = W.stride(0)).  An op other than 0 or 1
 * is B200_ERR_BAD_ARG.  (N, N) is b200_gemm_f32_ex / b200_gemm_bf16 / b200_gemm_s8s32 exactly: same kernels, kernel
 * names, launches and bits.  The (alpha, beta) rules of b200_gemm_f32_ex hold for every layout; AUTO picks its route
 * from m, n, k and the TMA-ability of the operands as stored, as for NN.  DEVICE pointers, asynchronous on `stream`.
 *
 * No operand is copied to row-major first where the tensor cores can read it as stored: wgmma reads 16-bit operands
 * K-major or MN-major, so A^T is staged as MN-major A and B^T as K-major B.  tf32 and int8 read only K-major
 * operands, so B^T is read in place and a transposed A (or, as for NN, a row-major B) goes through transpose_kernel
 * into the workspace.  Kernel launches per call (TMA-able operands):
 *
 *   path                    NN   NT (B^T given)   TN (A^T given)   TT
 *   bf16 -> fp32 / bf16      1   1                1                1     operands read in place
 *   fp16 -> fp32 / fp16      1   1                1                1     operands read in place (b200_gemm_f16_ex)
 *   bf16 / fp16 batched      1   1                1                1     every entry in one launch (_batched; also
 *                                                                        generic and alpha == 0 / k == 0: 1)
 *   bf16 / fp16 grouped      1   1                -                -     every group in one launch (_grouped; also
 *                                                                        generic and alpha == 0 / k == 0: 1)
 *   bf16 / fp16 grouped (K)  1   1                1                1     every group in one launch (_grouped_k; TN on
 *                                                                        the tensor cores, NN / NT / TT generic;
 *                                                                        alpha == 0 / total_k == 0: 1)
 *   TF32, int8               2   1                3                2     transposes into the workspace
 *   BF16X3, BF16X2           2   2                2                2     one split launch for both operands
 *   F16X2                    4   3                5                4     B^T's column maxima are its row maxima (the
 *                                                                        row pre-pass); A^T's row maxima are column
 *                                                                        maxima (column maxima + column split)
 *   STRICT                   1   2                2                3     A^T / B^T transposed into the workspace,
 *                                                                        then the unchanged FFMA kernel
 *   not TMA-able (generic)   1   1                1                1
 *
 * Every transposed result is bit-identical to the NN call on row-major copies of the operands: the planes, maxima and
 * transposes hold the same values and the MMAs take the same K order.  A new wgmma kernel is named with the layout
 * after the kind ("tc_bf16_nt_128x256", "tc_f16x2_tn_128x128"); a route that runs an NN kernel keeps its name.
 * Workspace: b200_gemm_workspace_bytes_op gives what the fp32 route uses (transposes and plane padding included; for
 * AUTO the largest of the routes AUTO may take at this size), equal to b200_gemm_workspace_bytes for (N, N).  bf16
 * uses none; int8 uses n * k16 bytes for a row-major B and m * k16 (at a 1 KB-aligned offset after B's) for a
 * transposed A, k16 = k rounded up to 16.  The packed handles, the row-panel plan, the requantising int8 GEMM and the
 * host-pointer entry points take row-major operands only. */
#define B200_OP_N 0   /* operand stored as is: op(A) = A (m x k, lda >= k); op(B) = B (k x n, ldb >= n)      */
#define B200_OP_T 1   /* operand stored transposed: A as k x m (lda >= m); B as n x k (ldb >= k), row-major */
int b200_gemm_f32_op(int op_a, int op_b, int m, int n, int k, float alpha,
                     const float* dA, int lda, const float* dB, int ldb, float beta,
                     float* dC, int ldc, int precision_mode, void* stream);
int b200_gemm_bf16_op(int op_a, int op_b, int m, int n, int k,
                      const uint16_t* dA, int lda, const uint16_t* dB, int ldb,
                      void* dC, int ldc, int out_type, void* stream);
int b200_gemm_s8s32_op(int op_a, int op_b, int m, int n, int k,
                       const int8_t* dA, int lda, const int8_t* dB, int ldb,
                       int32_t* dC, int ldc, void* stream);
size_t b200_gemm_workspace_bytes_op(int op_a, int op_b, int m, int n, int k, int precision_mode);

/* ---- FP8 tensor-core GEMM (torch._scaled_mm) ----------------------------------------------------------------------
 *   C = round_out( (acc * sa_i) * sb_j + bias_j )
 * acc is op(A) op(B) of the FP8 operands (raw bytes), op_a / op_b and lda / ldb as for the _op entry points; each step
 * is one fp32 round-to-nearest operation (no FMA contraction) and round_out one rounding to out_type (B200_OUT_F32,
 * _BF16 or _F16; fp16 overflows to +-inf).
 *   a_type / b_type: B200_FP8_E4M3 or B200_FP8_E5M2.  (e4m3, e4m3), (e4m3, e5m2) and (e5m2, e4m3) are supported, as in
 *     torch; (e5m2, e5m2) is B200_ERR_UNSUPPORTED.  e4m3 has NaN but no inf; e5m2 has both.  Non-finite operands and
 *     scales propagate as IEEE arithmetic does (0 * inf is NaN).
 *   dScaleA / dScaleB: fp32 on the device, never read by the host (no synchronisation; the call can be captured in a
 *     CUDA graph and the scales rewritten between replays).  scale_a_rowwise = 0: one element; 1: m elements, one per row
 *     of op(A).  scale_b_colwise = 0: one element; 1: n elements, one per column of op(B).  Any other flag is
 *     B200_ERR_BAD_ARG, and so is a null scale when there is work to do.
 *   dBias: null, or n elements of C's type (bf16 / fp16 bits, or fp32 for B200_OUT_F32), added after scaling.
 *   fast_accum = 0 (torch's default): every k-block of 128 elements starts a fresh tensor-core accumulator, added with a
 *     rounded fp32 add to the tile's running sum in registers; 128 x 128 tiles.  The tensor core keeps 14 significant
 *     bits when it adds FP8 products into its accumulator (measured on an H100 80GB HBM3 with crafted sums, DESIGN
 *     §4.7), so the error is bounded by that of 128-term chunks plus an fp32 running sum:
 *     |acc - exact| <= (8 * 2^-13 + ceil(k / 128) * 2^-24) * sum_k |a_k b_k|; measured on random e4m3 operands up to
 *     k = 16384: <= 4e-5 of sum |a b|, equal to torch._scaled_mm(use_fast_accum=False) on the same card.
 *     fast_accum = 1: one tensor-core accumulator over all of K (torch's use_fast_accum), 128 x 256 / 192 / 128 tiles;
 *     its error grows with K: measured 3.0e-4 to 3.9e-4 of sum |a b| for k = 1024 to 16384.
 * Any m, n, k; m == 0 or n == 0 is a no-op; k == 0 stores round_out(+0 + bias_j), or +0.  No K-split tail.  Every call
 * runs on the tensor cores: (N, T) with 16-byte aligned bases and pitches (torch's row-major A and column-major B) is
 * read in place; B given row-major and A given transposed are transposed into the workspace, and an operand whose base
 * or pitch is not a multiple of 16 bytes is copied there at a 16-byte pitch.  Every layout and pitch gives the bits of
 * the aligned (N, T) call.  Workspace: n * k16 bytes for B unless it is read in place, then m * k16 for A (at a 1 KB
 * aligned offset after B's) unless A is read in place, k16 = k rounded up to 16; reserve that much before the first
 * such call to keep it allocation-free.  Kernels: "tc_e4m3_obf16_128x256", "tc_e4m3e5m2_of32_acc_128x128", ... */
#define B200_FP8_E4M3 0
#define B200_FP8_E5M2 1
int b200_gemm_fp8(int op_a, int op_b, int a_type, int b_type, int m, int n, int k,
                  const uint8_t* dA, int lda, const uint8_t* dB, int ldb,
                  const float* dScaleA, int scale_a_rowwise, const float* dScaleB, int scale_b_colwise,
                  const void* dBias, void* dC, int ldc, int out_type, int fast_accum, void* stream);

/* ---- Blockwise-scaled FP8 GEMM (torch._scaled_mm's 1 x 128 / 128 x 128 scales, DeepSeek-V3's recipe) ---------------
 * K is cut into q = ceil(k / 128) k-blocks; block b covers K elements [128 b, 128 b + 128), the last one possibly
 * partial.  For each block, in order:
 *   acc_b(i, j)  the FP8 product over block b, a fresh tensor-core accumulator (b200_gemm_fp8's promoted chain)
 *   s_b(i, j)  = rn(sa_b(i) * sb_b(j))                  one fp32 multiply
 *   sum        = fma(acc_b(i, j), s_b(i, j), sum)       one fp32 fused multiply-add, from sum = +0
 * and C = round_out(rn(sum + bias_j)): the bias add and the output rounding of b200_gemm_fp8, no further scaling.
 *   dScaleA: fp32 on the device.  scale_a_block = 1: sa_b(i) = dScaleA[i * sa_row_stride + b * sa_kb_stride] (1 x 128:
 *     one scale per row and k-block); 128: sa_b(i) = dScaleA[(i / 128) * sa_row_stride + b * sa_kb_stride] (128 x 128).
 *   dScaleB: fp32 on the device.  scale_b_block = 1: sb_b(j) = dScaleB[b * sb_kb_stride + j * sb_col_stride] (1 x 128);
 *     128: sb_b(j) = dScaleB[b * sb_kb_stride + (j / 128) * sb_col_stride] (128 x 128).
 *   Strides are in elements, any value >= 0 (0 broadcasts; torch's outer-dim-major, row-major and padded layouts all
 *   work); the byte offset of the last scale read must fit a signed 64-bit integer.  The recipes are torch's three:
 *   (1, 128), (1, 1) and (128, 1); (128, 128) is B200_ERR_UNSUPPORTED.  Neither scale is read by the host: the call
 *   never synchronises and can be captured in a CUDA graph, with the scales rewritten between replays.
 * Operand pairs, output types, the bias, op_a / op_b, pitches, tails, m == 0 / n == 0 and k == 0 (round_out(+0 +
 * bias_j), no scale read), the non-finite rules and the routes (and so the workspace) are b200_gemm_fp8's; there is no
 * fast-accumulation form.  Every block size, stride and pointer is checked before the device is touched: a block size
 * other than 1 or 128, a negative stride, a null scale when m and n are nonzero or a last index out of range is
 * B200_ERR_BAD_ARG.
 * Error: each acc_b is within 8 * 2^-13 * sum_{k in b} |a_k b_k| of the exact block product (b200_gemm_fp8's 128-element
 * chunk bound); with the rounding of s_b and one fp32 rounding of each FMA,
 *   |sum - sum_b s_b exact_b| <= sum_b |s_b| (8 * 2^-13 + 2^-24) sum_{k in b} |a_k b_k| + q * 2^-24 * max_b |partial sum|.
 * On exact-class operands (each acc_b exact) the result is the fp32 chain above bit for bit.  Tiles are 128 x 128, six
 * stages, each stage's 128 + 128 scales staged in shared memory by the producer warpgroup.  Kernels:
 * "tc_e4m3_obf16_blk_128x128", "tc_e5m2e4m3_of32_blk_128x128", ... */
int b200_gemm_fp8_blockwise(int op_a, int op_b, int a_type, int b_type, int m, int n, int k,
                            const uint8_t* dA, int lda, const uint8_t* dB, int ldb,
                            const float* dScaleA, int scale_a_block, long long sa_row_stride, long long sa_kb_stride,
                            const float* dScaleB, int scale_b_block, long long sb_kb_stride, long long sb_col_stride,
                            const void* dBias, void* dC, int ldc, int out_type, void* stream);

/* ---- FP8 outputs of the FP8 GEMMs (torch._scaled_mm's scale_result; a fused 1 x 128 quantisation of C) ------------
 * Each element first gets the fp32 value v that b200_gemm_fp8 / b200_gemm_fp8_blockwise form before round_out:
 *   b200_gemm_fp8_q8:            v = act(rn(rn(rn(acc * sa_i) * sb_j) + bias_j))
 *   b200_gemm_fp8_blockwise_q8:  v = act(rn(sum + bias_j)), sum the blockwise FMA fold
 * dBiasBf16 is null (then -0 is added) or n bf16 values; act is a B200_ACT_* code, the fp32 activation of the 16-bit
 * epilogue.  c_type is B200_FP8_E4M3 (F = 448) or B200_FP8_E5M2 (F = 57344); C is m rows of ldc >= n bytes, any base
 * and any pitch.  fp8() below is round to nearest even with finite values past +-F saturated to +-F and NaN kept NaN.
 *   Static mode (dScaleC null): c_ij = fp8(rn(v_ij / s_r)), s_r = *dScaleResult (fp32 on the device, never read by the
 *     host), null = 1.  The rule is torch._scaled_mm's scale_result: torch's CPU kernel divides by it, and torch on CUDA
 *     saturates an FP8 output (measured with torch 2.11+cu128 on an H100 80GB HBM3; that build ignores scale_result on
 *     CUDA with tensorwise scales, so it equals this call only for s_r = 1.  DESIGN §9).
 *   Dynamic 1 x 128 mode (dScaleC non-null, dScaleResult must be null): for row i and column block c (columns
 *     [128 c, min(128 c + 128, n))), amax = max |v| over the block, d = rn(amax / F), d = 1 when that is 0, d = NaN when
 *     the block holds a NaN or an inf (all its elements are then NaN); c_ij = fp8(rn(v_ij / d)) and
 *     dScaleC[i * sc_row_stride + c * sc_blk_stride] = d.  (C, dScaleC) is then the (A, scale_a) of a following
 *     b200_gemm_fp8_blockwise call with scale_a_block = 1 and k = n.  The scale layout is row-major (m, q_n)
 *     (sc_blk_stride == 1, sc_row_stride >= q_n) or outer-dim-major (sc_row_stride == 1, sc_blk_stride >= m), q_n =
 *     ceil(n / 128), the stride of an extent-1 dimension being free; anything else is B200_ERR_BAD_ARG.
 * Everything else (operand pairs, input scales, op_a / op_b, pitches, routes and workspace, fast_accum, the argument
 * checks before the device is touched) is b200_gemm_fp8's / b200_gemm_fp8_blockwise's.  m == 0 or n == 0 is a no-op;
 * k == 0 quantises v = act(rn(+0 + bias_j)) in an element-wise pass that reads no operand and no input scale.  Tiles:
 * promoted 128 x 128, fast 128 x 256 or 128 x 128 (no 192-wide tile: it would split a 128-column block), blockwise
 * 128 x 128.  Kernels: "tc_e4m3_oe4m3_acc_128x128", "tc_e4m3e5m2_oe5m2_128x256", "tc_e4m3_oe4m3_blk_128x128", ... */
int b200_gemm_fp8_q8(int op_a, int op_b, int a_type, int b_type, int m, int n, int k,
                     const uint8_t* dA, int lda, const uint8_t* dB, int ldb,
                     const float* dScaleA, int scale_a_rowwise, const float* dScaleB, int scale_b_colwise,
                     const uint16_t* dBiasBf16, int act, int fast_accum, int c_type, uint8_t* dC, int ldc,
                     const float* dScaleResult, float* dScaleC, long long sc_row_stride, long long sc_blk_stride,
                     void* stream);
int b200_gemm_fp8_blockwise_q8(int op_a, int op_b, int a_type, int b_type, int m, int n, int k,
                               const uint8_t* dA, int lda, const uint8_t* dB, int ldb,
                               const float* dScaleA, int scale_a_block, long long sa_row_stride, long long sa_kb_stride,
                               const float* dScaleB, int scale_b_block, long long sb_kb_stride, long long sb_col_stride,
                               const uint16_t* dBiasBf16, int act, int c_type, uint8_t* dC, int ldc,
                               const float* dScaleResult, float* dScaleC, long long sc_row_stride,
                               long long sc_blk_stride, void* stream);

/* ---- Grouped and batched FP8 GEMMs (torch._scaled_grouped_mm 2-D x 3-D and 3-D x 3-D; FP8 mixture-of-experts layers) --
 * Every entry is one (N, T) b200_gemm_fp8 call with rowwise scales and no bias, all of them in one launch:
 *   C_e = round_out( (A_e B_e^T * sa_e[i]) * sb_e[j] )
 * A_e is row-major (lda >= k) and every B_e is stored n x k (ldb >= k): torch's column-major mat_b, the
 * W.transpose(-2, -1) of a (G, n, k) weight.  Operand pairs, output types, fast_accum, the non-finite rules and the
 * rounding are b200_gemm_fp8's, and so each entry's C is bit for bit that call's on the entry's rows, B and scales (the
 * same kernel code at the same tile width; b200_gemm_debug_set_bn forces a fast width for both).
 *   b200_gemm_fp8_grouped: group g is rows [end_{g-1}, end_g) of A (total_m x k) and C, times B_g = dB + g * stride_b,
 *     with the ends of b200_gemm_bf16_grouped (end_{-1} = 0, end_g = min(max(dOffs[g], end_{g-1}), total_m), read on
 *     the device; rows from end_{G-1} on are never written).  sa = dScaleA[row of A] (total_m elements), sb_g =
 *     dScaleB + g * scale_b_stride (n elements each).
 *   b200_gemm_fp8_batched: entry b is A_b = dA + b * stride_a (m x k), B_b = dB + b * stride_b, C_b = dC + b * stride_c,
 *     sa_b = dScaleA + b * scale_a_stride (m elements), sb_b = dScaleB + b * scale_b_stride (n elements).  A stride of
 *     0 broadcasts an operand; its scales still follow their own stride, so each entry may scale a shared A
 *     differently.  batch == 1 is the (N, T) b200_gemm_fp8 call with rowwise scales: same kernel, name and bits.
 * Scales are fp32 on the device and never read by the host, like the offsets: the calls never synchronise and can be
 * captured in a CUDA graph, with offsets and scales rewritten between replays.  No bias (torch refuses one here), no
 * workspace, no K-split tail.  k == 0 stores +0 over the covered rows / entries and reads no scale.
 * Argument rules, all checked before the device is touched: the types and flags of b200_gemm_fp8; the sizes, groups,
 * offsets, strides, overlap and tile-count bounds of b200_gemm_bf16_grouped / _batched, with the scale strides >= 0 and
 * bounded like the operand strides; a null scale (or offs) with work to do: B200_ERR_BAD_ARG.  The operands must be
 * read in place by the tensor cores: 16-byte aligned bases, lda, ldb and the operand strides multiples of 16 bytes, and
 * every input stride 0 or at least one entry (rows x ld); anything else is B200_ERR_UNSUPPORTED (there is no CUDA-core
 * FP8 kernel, and staging every entry's B would copy all of it).  Tiles are b200_gemm_fp8's: promoted 128 x 128, or
 * fast at pick_bn's width over the stack's tiles (a grouped call counts its bound of ceil(total_m / 128) + G tile rows).
 * Kernels: "tc_e4m3_obf16_grp_128x256", "tc_e4m3_of32_grp_acc_128x128", "tc_e4m3e5m2_of16_bat_128x192", ...; a k == 0
 * call runs "fill_zero_grp" / "fill_zero_bat". */
int b200_gemm_fp8_grouped(int a_type, int b_type, int total_m, int n, int k, const uint8_t* dA, int lda,
                          const uint8_t* dB, int ldb, long long stride_b, const int32_t* dOffs, int groups,
                          const float* dScaleA, const float* dScaleB, long long scale_b_stride,
                          void* dC, int ldc, int out_type, int fast_accum, void* stream);
int b200_gemm_fp8_batched(int a_type, int b_type, int m, int n, int k, const uint8_t* dA, int lda, long long stride_a,
                          const uint8_t* dB, int ldb, long long stride_b, const float* dScaleA, long long scale_a_stride,
                          const float* dScaleB, long long scale_b_stride, void* dC, int ldc, long long stride_c,
                          int batch, int out_type, int fast_accum, void* stream);

/* ---- Grouped and batched blockwise-scaled FP8 GEMMs (DeepSeek-V3-style FP8 mixture-of-experts layers) ---------------
 * Every entry is one (N, T) b200_gemm_fp8_blockwise call with no bias, all of them in one launch, and equals that call
 * on the entry's rows, B and scales bit for bit (the same MMA chain, fold and store):
 *   C_e = round_out(sum_e),  sum_e = fma(acc_b, rn(sa_b(i) * sb_b(j)), sum_e) over the k-blocks b in order, from +0.
 * A_e is row-major (lda >= k) and every B_e is stored n x k (ldb >= k), as for b200_gemm_fp8_grouped / _batched.
 *   b200_gemm_fp8_blockwise_grouped: group g is rows [end_{g-1}, end_g) of A (total_m x k) and C, times B_g = dB + g *
 *     stride_b, with b200_gemm_bf16_grouped's clamped ends read on the device (rows from end_{G-1} on are never
 *     written).  scale_a is always 1 x 128 (a 128-row block would straddle groups), indexed by the row of A:
 *     sa_b(i) = dScaleA[i * sa_row_stride + b * sa_kb_stride] (torch's (total_m, q) scale_a).  Group g's scale_b
 *     starts at dScaleB + g * scale_b_stride and is indexed as b200_gemm_fp8_blockwise's (scale_b_block 1 or 128).
 *   b200_gemm_fp8_blockwise_batched: entry e is A_e = dA + e * stride_a (m x k), B_e = dB + e * stride_b, C_e = dC + e
 *     * stride_c; its scales start at dScaleA + e * scale_a_stride and dScaleB + e * scale_b_stride and are indexed as
 *     b200_gemm_fp8_blockwise's, with any of its three recipes; (128, 128) is B200_ERR_UNSUPPORTED.  An operand stride
 *     of 0 broadcasts the operand; its scales still follow their own stride.  batch == 1 is the (N, T)
 *     b200_gemm_fp8_blockwise call with no bias: same kernel, name and bits.
 * Neither the offsets nor the scales are read by the host: the calls never synchronise and can be captured in a CUDA
 * graph.  No bias, no fast accumulation, no workspace, no K-split tail.  k == 0 stores +0 over the covered rows /
 * entries and reads no scale.  A scale row past an entry's rows (a grouped A's next group) and a column past n are
 * never read, whatever the offsets.
 * Argument rules, all checked before the device is touched: the types of b200_gemm_fp8; the block sizes (1 or 128),
 * strides (>= 0) and last-scale-index bound of b200_gemm_fp8_blockwise, that index including (G - 1) times the entry
 * stride; the sizes, groups, offsets, strides, overlap and tile bounds of b200_gemm_fp8_grouped / _batched, with the
 * scale entry strides bounded like the operand strides; a null scale (or offs) with work to do: B200_ERR_BAD_ARG.
 * Operands not read in place, as for b200_gemm_fp8_grouped / _batched: B200_ERR_UNSUPPORTED.  Tiles are 128 x 128,
 * six stages, as b200_gemm_fp8_blockwise's.  Kernels: "tc_e4m3_obf16_grp_blk_128x128", "tc_e5m2e4m3_of32_bat_blk_128x128",
 * ...; a k == 0 call runs "fill_zero_grp" / "fill_zero_bat". */
int b200_gemm_fp8_blockwise_grouped(int a_type, int b_type, int total_m, int n, int k,
                                    const uint8_t* dA, int lda, const uint8_t* dB, int ldb, long long stride_b,
                                    const int32_t* dOffs, int groups,
                                    const float* dScaleA, long long sa_row_stride, long long sa_kb_stride,
                                    const float* dScaleB, int scale_b_block, long long sb_kb_stride,
                                    long long sb_col_stride, long long scale_b_stride,
                                    void* dC, int ldc, int out_type, void* stream);
int b200_gemm_fp8_blockwise_batched(int a_type, int b_type, int m, int n, int k,
                                    const uint8_t* dA, int lda, long long stride_a,
                                    const uint8_t* dB, int ldb, long long stride_b,
                                    const float* dScaleA, int scale_a_block, long long sa_row_stride,
                                    long long sa_kb_stride, long long scale_a_stride,
                                    const float* dScaleB, int scale_b_block, long long sb_kb_stride,
                                    long long sb_col_stride, long long scale_b_stride,
                                    void* dC, int ldc, long long stride_c, int batch, int out_type, void* stream);

/* ---- FP8 outputs of the grouped and batched FP8 GEMMs (a fused 1 x 128 quantisation of each entry's C) -------------
 * Each call is its stacked parent above with the output type replaced by the dynamic 1 x 128 mode of b200_gemm_fp8_q8:
 * every group or entry's C and scales are bit for bit the (N, T) single-matrix call in dynamic mode with a null bias
 * and a null dScaleResult on the entry's rows, B and scales, at the same tile width:
 *   b200_gemm_fp8_grouped_q8 / _batched_q8:                      b200_gemm_fp8_q8,  v = act(rn(rn(rn(acc * sa_i) * sb_j) + -0))
 *   b200_gemm_fp8_blockwise_grouped_q8 / _blockwise_batched_q8:  b200_gemm_fp8_blockwise_q8,  v = act(rn(sum + -0))
 * then per row and 128-column block d = rn(amax / F) (1 when that is 0, NaN for a NaN or an inf in the block), c =
 * fp8(rn(v / d)), and d is stored.  act is a B200_ACT_* code, c_type B200_FP8_E4M3 or B200_FP8_E5M2; C is any base
 * and pitch (bytes = elements), as for b200_gemm_fp8_q8.
 *   Grouped: dScaleC is indexed by the row of C, dScaleC[i * sc_row_stride + c * sc_blk_stride] over (total_m, q_n),
 *     q_n = ceil(n / 128): exactly the (total_m, q) scale_a that b200_gemm_fp8_blockwise_grouped reads, so (C, dScaleC)
 *     is the next grouped blockwise GEMM's (A, scale_a).  Rows from end_{G-1} on are written neither in C nor in
 *     dScaleC.
 *   Batched: entry e's C starts at dC + e * stride_c and its scales at dScaleC + e * sc_entry_stride, each indexed as
 *     b200_gemm_fp8_q8's over (m, q_n).  batch == 1 is the single-matrix call itself: same kernel, name and bits.
 * Argument rules, all checked before the device is touched: the parent's, and c_type, act and the strides of
 * b200_gemm_fp8_q8; a null dScaleC with work to do; a scale layout that is neither row-major nor outer-dim-major over
 * (total_m, q_n) or (m, q_n) (b200_gemm_fp8_q8's rule); batch > 1 with sc_entry_stride below one entry's last scale
 * index + 1 (entries would overlap), above 2^60 / (batch - 1), or with a last index, entry term included, whose byte
 * offset does not fit a signed 64-bit integer: B200_ERR_BAD_ARG.  No bias, no static scale_result, no 128 x 128 output
 * blocks.  k == 0 stores act(+0) quantised (the FP8 +0 byte) and d = 1 over the covered rows or entries, reading no
 * operand and no scale; the grouped form finds its rows from the clamped offsets on the device.  The calls never
 * synchronise and can be captured in a CUDA graph.  Tiles: promoted 128 x 128, fast 128 x 256 or 128 x 128 (no
 * 192-wide tile), blockwise 128 x 128.  Kernels: "tc_e4m3_oe4m3_grp_128x256", "tc_e4m3e5m2_oe5m2_bat_acc_128x128",
 * "tc_e5m2e4m3_oe4m3_grp_blk_128x128", ...; a k == 0 call runs "fp8_q8_k0_grp" / "fp8_q8_k0_bat". */
int b200_gemm_fp8_grouped_q8(int a_type, int b_type, int total_m, int n, int k, const uint8_t* dA, int lda,
                             const uint8_t* dB, int ldb, long long stride_b, const int32_t* dOffs, int groups,
                             const float* dScaleA, const float* dScaleB, long long scale_b_stride, int act,
                             int fast_accum, int c_type, uint8_t* dC, int ldc, float* dScaleC, long long sc_row_stride,
                             long long sc_blk_stride, void* stream);
int b200_gemm_fp8_batched_q8(int a_type, int b_type, int m, int n, int k, const uint8_t* dA, int lda, long long stride_a,
                             const uint8_t* dB, int ldb, long long stride_b, const float* dScaleA,
                             long long scale_a_stride, const float* dScaleB, long long scale_b_stride, int act,
                             int fast_accum, int c_type, uint8_t* dC, int ldc, long long stride_c, float* dScaleC,
                             long long sc_row_stride, long long sc_blk_stride, long long sc_entry_stride, int batch,
                             void* stream);
int b200_gemm_fp8_blockwise_grouped_q8(int a_type, int b_type, int total_m, int n, int k,
                                       const uint8_t* dA, int lda, const uint8_t* dB, int ldb, long long stride_b,
                                       const int32_t* dOffs, int groups,
                                       const float* dScaleA, long long sa_row_stride, long long sa_kb_stride,
                                       const float* dScaleB, int scale_b_block, long long sb_kb_stride,
                                       long long sb_col_stride, long long scale_b_stride, int act, int c_type,
                                       uint8_t* dC, int ldc, float* dScaleC, long long sc_row_stride,
                                       long long sc_blk_stride, void* stream);
int b200_gemm_fp8_blockwise_batched_q8(int a_type, int b_type, int m, int n, int k,
                                       const uint8_t* dA, int lda, long long stride_a,
                                       const uint8_t* dB, int ldb, long long stride_b,
                                       const float* dScaleA, int scale_a_block, long long sa_row_stride,
                                       long long sa_kb_stride, long long scale_a_stride,
                                       const float* dScaleB, int scale_b_block, long long sb_kb_stride,
                                       long long sb_col_stride, long long scale_b_stride, int act, int c_type,
                                       uint8_t* dC, int ldc, long long stride_c, float* dScaleC,
                                       long long sc_row_stride, long long sc_blk_stride, long long sc_entry_stride,
                                       int batch, void* stream);

/* ---- Blockwise FP8 quantisers (the operands of the blockwise FP8 GEMMs, with an optional transposed copy) ----------
 * x is batch entries of a rows x cols row-major matrix of in_type (B200_OUT_F32, B200_OUT_BF16 or B200_OUT_F16 used as
 * element-type codes), entry b at dX + b * stride_x with row pitch ldx >= cols elements, any base and any pitch.  Per
 * block, amax = max |x| over the block's elements inside the matrix (NaN if one is NaN), and with F = 448 (c_type
 * B200_FP8_E4M3) or 57344 (B200_FP8_E5M2):
 *   d = rn(amax / F), 1 when that is 0, NaN when the block holds a NaN or an inf;   q = fp8(rn(x / d))
 * fp8() round to nearest even with finite values saturated to +-F and NaN kept: exactly the dynamic 1 x 128 rule of
 * b200_gemm_fp8_q8, whose (C, dScaleC) equals this call on its fp32 C.  Every input converts to fp32 exactly.
 *   block = 1 (1 x 128: activations, gradients): one d per row i and 128-column block c, at dScale[i * s_row + c * s_blk]
 *     over (rows, ceil(cols / 128)).  With dQt non-null, dQt (cols x rows, pitch ldqt >= rows bytes) is the 1 x 128
 *     quantisation of x^T: dQt[j * ldqt + i] = fp8(rn(x[i, j] / dt)), dt = dScaleT[j * st_row + (i / 128) * st_blk]
 *     over (cols, ceil(rows / 128)), one per column of x and 128-row block.  dScaleT is required with dQt.
 *   block = 128 (128 x 128: weights): one d per 128 x 128 block (edge blocks clipped) at dScale[r * s_row + c * s_blk]
 *     over (ceil(rows / 128), ceil(cols / 128)).  With dQt non-null, dQt is q^T byte for byte and shares the scales
 *     (dScale transposed): dScaleT must be null.
 * dQ holds q, rows x cols bytes at pitch ldq >= cols.  Entry b's q, scales, qt and transposed scales start at dQ + b *
 * stride_q, dScale + b * s_entry, dQt + b * stride_qt and dScaleT + b * st_entry.  Nothing outside the matrices and
 * their scale entries is written.  (q, dScale) with block = 1 is b200_gemm_fp8_blockwise's (A, scale_a) with
 * scale_a_block = 1; with block = 128 it is a weight W (n x k) whose (B^T, scale_b^T) take scale_b_block = 128.
 * rows == 0, cols == 0 or batch == 0 is a no-op, null pointers included.  One launch, no workspace, no host
 * synchronisation: the call can be captured in a CUDA graph.
 * Argument rules, all checked before the device is touched (B200_ERR_BAD_ARG): the type codes and block; negative
 * sizes or strides; ldx, ldq or (with dQt) ldqt below its minimum; a null dX, dQ or dScale, or a dScaleT that is not
 * given exactly with dQt (1 x 128) or is given (128 x 128); a scale layout that is neither row-major nor outer-dim-major
 * (b200_gemm_fp8_q8's rule for dScaleC, the stride of an extent-1 dimension being free); batch > 1 with an output
 * entry stride at or below its entry's last index (entries would overlap) or any entry stride above 2^60 / (batch - 1);
 * a last element of any tensor whose byte offset does not fit a signed 64-bit integer.
 * Kernels: "fp8_quant_bf16_e4m3_1x128", "fp8_quant_t_f32_e5m2_128x128", ... (_t: the transposed output is written). */
int b200_fp8_quantize(int in_type, int c_type, int block, int rows, int cols, int batch,
                      const void* dX, int ldx, long long stride_x,
                      uint8_t* dQ, int ldq, long long stride_q,
                      float* dScale, long long s_row, long long s_blk, long long s_entry,
                      uint8_t* dQt, int ldqt, long long stride_qt,
                      float* dScaleT, long long st_row, long long st_blk, long long st_entry, void* stream);

/* Pre-split operands for the split-precision modes (AUTO = the library default): the reference
 * leaves its "packAB interface open" for callers that reuse one operand (README.md:85; PackMatrixA/B,
 * aarch64/MMult_4x4_13.cpp:259,361).  TMA needs no repacking of row-major operands, but the fp32 ->
 * plane split is per-call work (the pre-pass) that a constant operand can pay once.
 *   b200_gemm_f32_pack_b   splits the k x n matrix B (F16X2, BF16X3, BF16X2) into a handle that owns its
 *                          device memory;
 *   b200_gemm_f32_pack_a   does the same for the m x k matrix A (F16X2 only);
 *   b200_gemm_f32_packed   computes C = A*B (accumulate = 0) or C += A*B (1) from fp32 A and packed B and
 *                          is bit-identical to b200_gemm_f32 / b200_gemm_f32_acc in the handle's mode;
 *   b200_gemm_f32_packed_ab  uses both handles and multiplies columns [a_k0, a_k0 + k) of packed A
 *                          (a_k0 a multiple of 8) by a packed B of exactly k rows: a K-sliced consumer
 *                          (B arriving in row blocks over NVLink) splits A once and each block of B as
 *                          it lands.
 * DEVICE pointers; a handle may be used by any number of later calls (stream-ordered after the pack
 * call) on the device it was made on and is released with b200_gemm_f32_pack_free / _free_a.  Modes
 * without a split (STRICT, TF32) return B200_ERR_UNSUPPORTED. */
typedef struct b200_packed_b b200_packed_b;
typedef struct b200_packed_a b200_packed_a;
int b200_gemm_f32_pack_b(int k, int n, const float* dB, int ldb, int precision_mode,
                         b200_packed_b** out, void* stream);
int b200_gemm_f32_pack_a(int m, int k, const float* dA, int lda, int precision_mode,
                         b200_packed_a** out, void* stream);
int b200_gemm_f32_packed(int m, int n, int k, const float* dA, int lda,
                         const b200_packed_b* packedB, float* dC, int ldc,
                         int accumulate, void* stream);
int b200_gemm_f32_packed_ab(int m, int n, int k, const b200_packed_a* packedA, int a_k0,
                            const b200_packed_b* packedB, float* dC, int ldc,
                            int accumulate, void* stream);
void b200_gemm_f32_pack_free(b200_packed_b* packedB);
void b200_gemm_f32_pack_free_a(b200_packed_a* packedA);

/* int8 x int8 -> int8 with the requantising tail of chgemm's kernels fused into the
 * GEMM epilogue (aarch64-int8/int8kernel_m4.S:386-426; signature :40):
 *   C(i,j) = sat_int8( round_ties_away( float(sum_p A(i,p)*B(p,j)) * dScales[i] (+ dBias[i]) ) )
 * int32 -> fp32 conversion rounds to nearest even, the multiply and the add round
 * separately (fmul, fadd), NaN converts to 0.  dScales has m entries, dBias has m
 * entries or is NULL (the kernel's `cmp bias, #0`).  C is written once as int8
 * (1 byte per element instead of 4).  DEVICE pointers; ldc in elements (bytes). */
int b200_gemm_s8s8_requant(int m, int n, int k,
                           const int8_t* dA, int lda, const int8_t* dB, int ldb,
                           int8_t* dC, int ldc, const float* dScales,
                           const float* dBias, void* stream);

/* ---- multi-GPU: C sharded by row panels, one exchange step (BASELINE config 5; SURVEY §8e) ------------
 * The reference has no multi-GPU code; north_star asks for "row-panels across the box's GPUs with one
 * NCCL broadcast of B over NVLink" behind this C ABI.  One process (or host thread) per GPU; rank i owns
 * A_i (m_local x k) and C_i (m_local x n); B (k x n) is valid on `root` before the call and on every rank
 * after it.  B crosses NVLink as K-slices (contiguous row blocks of the row-major operand, broadcast in
 * place with ncclBroadcast on the plan's own stream); A_i is split into its planes while the first slice
 * travels and slice j is multiplied while slices j+1.. are in flight.  Timing convention of the
 * reference's harness: operands resident, the exchange inside the call (cuda/test_MMult.cpp:84-112).
 *
 * NCCL is resolved with dlopen at first use (the libnccl.so.2 already loaded in the process, e.g. torch's,
 * else the system one; b200_nccl_load(path) forces one): libb200gemm.so itself does not link NCCL.
 *   nccl_comm   an ncclComm_t (as void*): the caller's own (torch: ProcessGroupNCCL._comm_ptr()) or one
 *               made with b200_comm_unique_id + b200_comm_init_rank (rank 0 creates the 128-byte id and
 *               hands it to the other ranks by whatever means the host has).  NULL = single rank.
 *   slice_rows  rows of B per K-slice (sum k, every boundary a multiple of 8), or NULL / n_slices 0 for the
 *               default (one slice on one rank; two slices weighted 1:3 up to 256 MB of B; equal ~256 MB slices, at most 8, beyond).
 * The plan owns all scratch (planes, events, streams): the compute calls never allocate. */
typedef struct b200_rowpanel b200_rowpanel;
int  b200_nccl_load(const char* libnccl_path_or_null);
const char* b200_nccl_last_error(void);
int  b200_comm_unique_id(void* id128);
int  b200_comm_init_rank(void** nccl_comm_out, const void* id128, int rank, int world);
int  b200_comm_destroy(void* nccl_comm);
int  b200_rowpanel_create(b200_rowpanel** out, void* nccl_comm, int m_local_max, int n, int k,
                          int precision_mode, const int* slice_rows, int n_slices);
void b200_rowpanel_destroy(b200_rowpanel* plan);
/* Tuning.  While a later K-slice is still being broadcast, the GEMM of the current slice shares the GPU with NCCL's
 * copy kernels.  Their tensor-core kernels then launch `sms` fewer CTAs than the device has SMs (default 0; ignored
 * unless more than 2 SMs stay in use), and the tiles are handed out round robin over the smaller grid.  sms = -1 is accepted and
 * changes nothing. */
int  b200_rowpanel_set_reserve_sms(b200_rowpanel* plan, int sms);
/* Diagnostics: with tracing on, timing events bracket every stage of a call; the dump synchronises the device and
 * writes, in ms after the call began: A split done, then per K-slice {broadcast begin, broadcast end, slice visible
 * on the compute stream, split done, GEMM done}.  Returns the number of values. */
void b200_rowpanel_trace(b200_rowpanel* plan, int enable);
int  b200_rowpanel_trace_dump(b200_rowpanel* plan, float* out_ms, int cap);
/* K-slice boundaries of the plan: writes min(n_slices + 1, cap) row offsets, returns n_slices. */
int  b200_rowpanel_slices(const b200_rowpanel* plan, int* bounds, int cap);
/* C_local = A_local * B on DEVICE pointers (dB: the operand on root, the receive buffer elsewhere; ldb == n
 * unless single-rank).  Asynchronous on `stream`. */
int  b200_gemm_f32_rowpanel(b200_rowpanel* plan, int m_local, int n, int k,
                            const float* dA_local, int lda, float* dB, int ldb,
                            float* dC_local, int ldc, int root, void* stream);
/* C_local += A_local * B with HOST pointers (the 9-arg MY_MMult contract, aarch64/MMult0.cpp:3-23, sharded):
 * B is read on root only; H2D, exchange, math and D2H are pipelined inside; synchronous. */
int  b200_gemm_f32_rowpanel_host(b200_rowpanel* plan, int m_local, int n, int k,
                                 const float* A_local, int lda, const float* B, int ldb,
                                 float* C_local, int ldc, int root);

/* ---- the 4-bit path (SURVEY §8 f-4) ------------------------------------------------------------------
 * The reference lists a cuda-int4 back-end and ships only the word "WIP" (cuda-int4/README.md:1;
 * README.md:13-15,118-120), so there is no interface to mirror: this is the chgemm idea (quantised operands,
 * wide accumulate) on OCP MXFP4 — E2M1 elements with one power-of-two UE8M0 scale per 32 consecutive K
 * elements, fp32 accumulate and output.  sm_90 has no 4-bit tensor-core operand: the GEMM expands both operands
 * exactly to bf16 (workspace) and runs the bf16 tensor-core kernel.
 *   quantize_a   A (m x k fp32, row-major)  -> dQ (m rows of kpad/2 bytes, two elements per byte, low nibble
 *                first; kpad = k rounded up to 128) + dSF (scale atoms, b200_mxf4_sf_bytes(m, k) bytes)
 *   quantize_b   B (k x n fp32, row-major)  -> B^T quantised along K: dQ has n rows (4-bit operands must be
 *                K-major for the tensor core: the one transposing pass of this library) + dSF(n, k)
 *   gemm_mxf4    C (m x n fp32) = dequant(A) * dequant(B)
 * Scale atom layout: [rows/128][kpad/128][512 bytes], byte (r%32)*16 + ((r/32)%4)*4 + (kblock%4).
 * DEVICE pointers, 16-byte aligned; asynchronous on `stream`. */
size_t b200_mxf4_q_bytes(int rows, int k);
size_t b200_mxf4_sf_bytes(int rows, int k);
int b200_mxf4_quantize_a(int m, int k, const float* dA, int lda, uint8_t* dQ, uint8_t* dSF, void* stream);
int b200_mxf4_quantize_b(int k, int n, const float* dB, int ldb, uint8_t* dQ, uint8_t* dSF, void* stream);
int b200_gemm_mxf4(int m, int n, int k, const uint8_t* dAq, const uint8_t* dSFA,
                   const uint8_t* dBq, const uint8_t* dSFB, float* dC, int ldc, void* stream);

/* Element-wise helper the bf16 config needs on the device: round-to-nearest-
 * even fp32 -> bf16 (the rounding SURVEY §8d prescribes for config 3 inputs). */
int b200_convert_f32_to_bf16(const float* dSrc, uint16_t* dDst, size_t count,
                             void* stream);

/* Test/diagnostic hook: overrides for the wgmma shared-memory descriptor (LBO, SBO) of the
 * MN-major B operand of the 16-bit kinds (bytes; 0 = library default). */
void b200_gemm_debug_set_b_desc(int lbo_bytes, int sbo_bytes);
/* Tuning hook: 0 = launch without programmatic dependent launch (default 1: the library's tensor-core and
 * pre-pass kernels are launched with the programmatic-serialisation attribute and order themselves with
 * griddepcontrol.wait, so a kernel's prologue overlaps the tail of its predecessor in the stream). */
void b200_gemm_debug_set_pdl(int mask);   /* bit 0: PDL on; bit 1: keep the F16X2 pre-pass of B on the caller's stream (default: auxiliary stream beside A's) */
/* Accepted for ABI compatibility; no effect (the sm_90 kernels use one static round-robin tile schedule). */
void b200_gemm_debug_set_dynamic_sched(int on);
/* Tuning hook: force the tensor-core tile width (128, 192 or 256; 0 = built-in heuristic). */
void b200_gemm_debug_set_bn(int bn);
/* Accepted for ABI compatibility; no effect (the sm_90 kernels have no CTA pairs). */
void b200_gemm_debug_set_cta_group(int cg);
/* Tuning hook: 1 (default) = the last partial round of tiles is split along K across the idle
 * CTAs and folded into C in order; 0 = whole tiles only. */
void b200_gemm_debug_set_split_tail(int on);
/* Test hook: the work schedule of the last tensor-core GEMM launch issued by the calling thread.  tiles: output
 * tiles of the launch (of every entry for a batched call); split: K parts of each tile of the last partial round
 * (1 = whole tiles only); full_tiles: tiles computed whole; ctas: the persistent grid.  Any pointer may be NULL. */
void b200_gemm_debug_last_schedule(int* tiles, int* split, int* full_tiles, int* ctas);
/* Tuning hook: K extent the tensor core accumulates before the epilogue folds the partial sum
 * into C with a rounded fp32 add (two-level accumulation of the split modes); 0 = whole K.
 * bf16x2_k sets both BF16X2 and F16X2.  A negative value restores the built-in default of its
 * mode(s): 512 for BF16X3 and BF16X2, 1024 for F16X2. */
void b200_gemm_debug_set_split_chunk(int bf16x3_k, int bf16x2_k);
/* Tuning hook: rows of A per raster group of the persistent tile schedule (0 = 2048). */
void b200_gemm_debug_set_group_rows(int rows);
/* Tuning hook for the strict fp32 kernels: bit 0 = half tiles in the last partial round (default on),
 * bit 1 = force the 128x256 fat-thread kernel; a negative value restores selection by size. */
void b200_gemm_debug_set_ffma_variant(int v);
/* Accepted for ABI compatibility; no effect (the sm_90 kernels have one epilogue form). */
void b200_gemm_debug_set_epilogue(int mask);
/* Measurement hook: while enabled, a CUDA-event pair is recorded on the launching stream around
 * every dominant GEMM kernel launch (not the split pre-pass).  b200_gemm_debug_kernel_time_ms
 * synchronises those events, stores the summed kernel time and returns the number of launches
 * covered (then resets).  bench.py's roofline.achieved comes from here. */
void b200_gemm_debug_kernel_timing(int enable);
int  b200_gemm_debug_kernel_time_ms(double* sum_ms);

#ifdef __cplusplus
}
#endif
#endif /* B200GEMM_H_ */
