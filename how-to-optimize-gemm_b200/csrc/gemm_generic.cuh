// gemm_generic.cuh — shape/stride-agnostic CUDA-core kernels (still GPU; there is no CPU path).
//
// They serve what TMA cannot describe: leading dimensions or base pointers that are not 16-byte
// aligned (TMA needs ld*sizeof % 16 == 0), and degenerate sizes.  The reference's hand kernels
// simply assume m,n % 128 == 0 and ignore lda/ldb/ldc (cuda/MMult_cuda_12.cu:231-234); chgemm's
// headline feature is that it does not (aarch64-int8/int8kernel_m4.S:62-93).  Sequential-k
// accumulation, so the fp32 instance keeps the strict contract of gemm_ffma.cuh.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <type_traits>

#include "ptx.cuh"

namespace b200 {

// Element types: float, int8_t, uint16_t = bf16 bits, __half = fp16.  Every 16-bit load is exact in fp32.
template <typename T> struct LoadAs;
template <> struct LoadAs<float>   { using Acc = float;   __device__ static float   ld(const float* p)   { return *p; } };
template <> struct LoadAs<int8_t>  { using Acc = int32_t; __device__ static int32_t ld(const int8_t* p)  { return (int32_t)*p; } };
template <> struct LoadAs<uint16_t>{ using Acc = float;   __device__ static float   ld(const uint16_t* p){ return __uint_as_float((uint32_t)*p << 16); } };
template <> struct LoadAs<__half>  { using Acc = float;   __device__ static float   ld(const __half* p)  { return __half2float(*p); } };

// fp32 -> 16-bit stores round to nearest even (fp16: beyond 65504 to +-inf)
template <typename Acc, typename OutT> __device__ __forceinline__ void store_out(OutT* p, Acc v);
template <> __device__ __forceinline__ void store_out<float, float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void store_out<int32_t, int32_t>(int32_t* p, int32_t v) { *p = v; }
template <> __device__ __forceinline__ void store_out<float, uint16_t>(uint16_t* p, float v) {
  *p = __bfloat16_as_ushort(__float2bfloat16_rn(v));
}
template <> __device__ __forceinline__ void store_out<float, __half>(__half* p, float v) { *p = __float2half_rn(v); }

// act(t + b) with a runtime activation code (EpiAct); b = -0 stands for no bias (t + -0 is t, zeros included).
__device__ __forceinline__ float act_bias(float t, float b, int act) {
  t = __fadd_rn(t, b);
  switch (act) {
    case ACT_RELU: return epi_act<ACT_RELU>(t);
    case ACT_GELU: return epi_act<ACT_GELU>(t);
    case ACT_GELU_TANH: return epi_act<ACT_GELU_TANH>(t);
    default: return t;
  }
}

// 64x64 tile, 256 threads, 4x4 per thread, BK = 16.
// Element strides per index: A(i, p) = A[i * a_rs + p * a_cs], B(p, j) = B[p * b_rs + j * b_cs].  Row-major A is
// (lda, 1), a transposed one (A^T stored k x m, pitch lda) is (1, lda); likewise B.  The arithmetic does not
// depend on the strides.
// axpby (fp32, bf16 or fp16 in; fp32 or 16-bit out): C = alpha * (A*B) + beta * C (b200_gemm_f32_ex, _bf16_ex,
// _f16_ex); the chains start from zero, alpha * chain is rounded, then fma(beta, float(C), .), rounded once more to
// a 16-bit C, and C is read only when beta != 0.
// bias / act (16-bit operands, b200_gemm_bf16_epi / _f16_epi; needs axpby): after the alpha / beta step, t + bias[j]
// (skipped for a null bias) goes through epi_act (ptx.cuh), the tensor-core kernel's activation.  act = -1: none.
// WALK_Y: a block computes the row blocks blockIdx.y, + gridDim.y, ... (launched when M needs more than gridDim.y's
// 65535 blocks).  Without it a block computes row block blockIdx.y only: a loop back-edge alone raises the 16-bit
// kernels from 40 registers to as many as 63, which would cost them occupancy on every call.
template <typename InT, typename OutT, bool WALK_Y = false>
__global__ void __launch_bounds__(256)
gemm_generic_kernel(int M, int N, int K, const InT* __restrict__ A, long long a_rs, long long a_cs,
                    const InT* __restrict__ B, long long b_rs, long long b_cs, OutT* __restrict__ C, long long ldc,
                    int accumulate, const float* __restrict__ rq_scale = nullptr,
                    const float* __restrict__ rq_bias = nullptr, int axpby = 0, float alpha = 1.f, float beta = 0.f,
                    const InT* __restrict__ bias = nullptr, int act = -1) {
  using Acc = typename LoadAs<InT>::Acc;
  __shared__ Acc As[16][64 + 4];
  __shared__ Acc Bs[16][64 + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int n0 = blockIdx.x * 64, mblocks = (int)(((long long)M + 63) / 64);
  // With WALK_Y, the k loop's closing __syncthreads (K > 0) orders one row block's last reads of As / Bs before the
  // next one's loads.
  for (int mb = blockIdx.y; mb < mblocks; mb += gridDim.y) {
    const int m0 = mb * 64;
    Acc acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
      for (int j = 0; j < 4; j++) acc[i][j] = 0;
    if constexpr (std::is_same<Acc, OutT>::value) {
      if (accumulate) {          // chain starts from C(i,j): the CPU harness contract C += A*B
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) {
            const int gm = m0 + ty + 16 * i, gn = n0 + tx + 16 * j;
            if (gm < M && gn < N) acc[i][j] = C[(long long)gm * ldc + gn];
          }
      }
    }

    for (int k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const int idx = threadIdx.x + r * 256;          // 0..1023
        const int am = idx >> 4, ak = idx & 15;          // A tile 64 x 16, k fastest
        const int gm = m0 + am, gk = k0 + ak;
        As[ak][am] = (gm < M && gk < K) ? LoadAs<InT>::ld(A + (long long)gm * a_rs + (long long)gk * a_cs) : (Acc)0;
        const int bk = idx >> 6, bn = idx & 63;          // B tile 16 x 64, n fastest
        const int gk2 = k0 + bk, gn = n0 + bn;
        Bs[bk][bn] = (gk2 < K && gn < N) ? LoadAs<InT>::ld(B + (long long)gk2 * b_rs + (long long)gn * b_cs) : (Acc)0;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < 16; kk++) {
        Acc a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; i++) a[i] = As[kk][ty + 16 * i];
#pragma unroll
        for (int j = 0; j < 4; j++) b[j] = Bs[kk][tx + 16 * j];
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) {
            if constexpr (sizeof(Acc) == 4 && !std::is_same<Acc, int32_t>::value)
              acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
            else
              acc[i][j] += a[i] * b[j];
          }
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int gm = m0 + ty + 16 * i;
      if (gm >= M) continue;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int gn = n0 + tx + 16 * j;
        if (gn < N) {
          if constexpr (std::is_same<OutT, int8_t>::value && std::is_same<Acc, int32_t>::value) {
            // requantising store (int8 C): per-row scale and optional per-row bias
            C[(long long)gm * ldc + gn] = (int8_t)requant_s8(acc[i][j], rq_scale[gm], rq_bias ? rq_bias[gm] : 0.0f,
                                                              rq_bias != nullptr);
          } else if constexpr (std::is_same<Acc, float>::value) {        // fp32, bf16 or fp16 C
            float v = acc[i][j];
            if (axpby) {
              v *= alpha;
              if (beta != 0.f) v = fmaf(beta, LoadAs<OutT>::ld(C + (long long)gm * ldc + gn), v);
            }
            if constexpr (sizeof(InT) == 2) {
              if (act >= 0) v = act_bias(v, bias != nullptr ? LoadAs<InT>::ld(bias + gn) : -0.f, act);
            }
            store_out<float, OutT>(C + (long long)gm * ldc + gn, v);
          } else {
            store_out<Acc, OutT>(C + (long long)gm * ldc + gn, acc[i][j]);
          }
        }
      }
    }
    if constexpr (!WALK_Y) break;
  }
}

// ---- small element-wise helpers ------------------------------------------------------------
__global__ void convert_f32_to_bf16_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst,
                                           size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) dst[i] = __bfloat16_as_ushort(__float2bfloat16_rn(src[i]));
}

// C = s * C over an m x n window (C = beta * C of the general epilogue when alpha == 0 or k == 0); 16-bit C is
// read exactly and the product rounded once
template <typename T>
__global__ void scale_inplace_kernel(int M, int N, T* __restrict__ C, long long ldc, float s) {
  for (int r = blockIdx.y; r < M; r += gridDim.y)
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < N; c += gridDim.x * blockDim.x) {
      T* e = C + (long long)r * ldc + c;
      store_out<float, T>(e, s * LoadAs<T>::ld(e));
    }
}

// C = act(beta * C + bias[c]) over an m x n window (the bias / activation epilogue when alpha == 0 or k == 0): beta == 0
// contributes +0 and leaves C unread; a null bias adds nothing.  16-bit C is read exactly and the result rounded once.
template <typename T, typename BiasT>
__global__ void bias_act_inplace_kernel(int M, int N, T* __restrict__ C, long long ldc, float s,
                                        const BiasT* __restrict__ bias, int act) {
  for (int r = blockIdx.y; r < M; r += gridDim.y)
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < N; c += gridDim.x * blockDim.x) {
      T* e = C + (long long)r * ldc + c;
      const float t = s != 0.f ? s * LoadAs<T>::ld(e) : 0.f;
      store_out<float, T>(e, act_bias(t, bias != nullptr ? LoadAs<BiasT>::ld(bias + c) : -0.f, act));
    }
}

template <typename T>
__global__ void fill_zero_kernel(int M, int N, T* __restrict__ C, long long ldc) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  for (int i = blockIdx.y; i < M; i += gridDim.y) C[(long long)i * ldc + j] = (T)0;
}

// ---- stacked 16-bit forms: strided batch and grouped -----------------------------------------------------------
// Kernels of their own, so that the single-matrix kernels above keep their code exactly.

// gemm_generic_kernel's tile for 16-bit operands with the alpha / beta epilogue (no accumulate, requant, bias or
// activation) at (m0, n0) of one M x N matrix: the same loads, the same fmaf chain in k order and the same store, so
// every matrix of a stacked call equals the 2-D generic call on that matrix bit for bit.  Every thread of the block
// calls it; it ends in __syncthreads (K > 0), so the block may call it again for another tile.  As / Bs are the
// calling kernel's own shared arrays: static __shared__ arrays here would be module-scope symbols shared by several
// kernels, and that alone changes the code ptxas emits for the unrelated 2-D generic kernels.
typedef float GenericTile[16][64 + 4];
template <typename InT, typename OutT>
__device__ __forceinline__ void generic_tile16(GenericTile& As, GenericTile& Bs, int m0, int n0, int M, int N, int K,
                                               const InT* __restrict__ A, long long a_rs, long long a_cs,
                                               const InT* __restrict__ B, long long b_rs, long long b_cs,
                                               OutT* __restrict__ C, long long ldc, int axpby, float alpha, float beta) {
  static_assert(sizeof(InT) == 2, "stacked generic kernels: 16-bit operands");
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += 16) {
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int idx = threadIdx.x + r * 256;
      const int am = idx >> 4, ak = idx & 15;
      const int gm = m0 + am, gk = k0 + ak;
      As[ak][am] = (gm < M && gk < K) ? LoadAs<InT>::ld(A + (long long)gm * a_rs + (long long)gk * a_cs) : 0.f;
      const int bk = idx >> 6, bn = idx & 63;
      const int gk2 = k0 + bk, gn = n0 + bn;
      Bs[bk][bn] = (gk2 < K && gn < N) ? LoadAs<InT>::ld(B + (long long)gk2 * b_rs + (long long)gn * b_cs) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; kk++) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; i++) a[i] = As[kk][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; j++) b[j] = Bs[kk][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();                                   // also orders this tile's last reads before the next tile's loads
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int gm = m0 + ty + 16 * i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int gn = n0 + tx + 16 * j;
      if (gn < N) {
        float v = acc[i][j];
        if (axpby) {
          v *= alpha;
          if (beta != 0.f) v = fmaf(beta, LoadAs<OutT>::ld(C + (long long)gm * ldc + gn), v);
        }
        store_out<float, OutT>(C + (long long)gm * ldc + gn, v);
      }
    }
  }
}

// Strided batch: entry z of each operand at X + z * x_bs (elements; 0 broadcasts A or B), the entries over
// blockIdx.z, gridDim.z at a time, and the row blocks over blockIdx.y, gridDim.y at a time.
template <typename InT, typename OutT>
__global__ void __launch_bounds__(256)
gemm_generic_batched_kernel(int batch, int M, int N, int K, const InT* __restrict__ A, long long a_rs, long long a_cs,
                            long long a_bs, const InT* __restrict__ B, long long b_rs, long long b_cs, long long b_bs,
                            OutT* __restrict__ C, long long ldc, long long c_bs, int axpby, float alpha, float beta) {
  __shared__ GenericTile As, Bs;
  const int mblocks = (int)(((long long)M + 63) / 64);
  for (int z = blockIdx.z; z < batch; z += gridDim.z)
    for (int mb = blockIdx.y; mb < mblocks; mb += gridDim.y)
      generic_tile16(As, Bs, mb * 64, blockIdx.x * 64, M, N, K, A + z * a_bs, a_rs, a_cs, B + z * b_bs, b_rs, b_cs,
                     C + z * c_bs, ldc, axpby, alpha, beta);
}

// scale_inplace_kernel (s != 0) and fill_zero_kernel (s == 0) over every entry: the k == 0 / alpha == 0 pass.
template <typename T>
__global__ void scale_inplace_batched_kernel(int batch, int M, int N, T* __restrict__ C, long long ldc, long long c_bs,
                                             float s) {
  for (int z = blockIdx.z; z < batch; z += gridDim.z)
    for (int r = blockIdx.y; r < M; r += gridDim.y)
      for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < N; c += gridDim.x * blockDim.x) {
        T* e = C + z * c_bs + (long long)r * ldc + c;
        store_out<float, T>(e, s * LoadAs<T>::ld(e));
      }
}
template <typename T>
__global__ void fill_zero_batched_kernel(int batch, int M, int N, T* __restrict__ C, long long ldc, long long c_bs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  for (int z = blockIdx.z; z < batch; z += gridDim.z)
    for (int i = blockIdx.y; i < M; i += gridDim.y) C[z * c_bs + (long long)i * ldc + j] = (T)0;
}

// Grouped: group g is rows [end[g], end[g + 1]) of one stacked row-major A (total_m x k, pitch lda) and C, times B_g
// at B + g * b_gs (group_table, ptx.cuh, clamps the offsets).  The tiles are 64-row blocks that each lie inside one
// group: blockIdx.x counts the blocks of every group in order (surplus blocks exit), blockIdx.y the column blocks,
// gridDim.y at a time.
template <typename InT, typename OutT>
__global__ void __launch_bounds__(256)
gemm_generic_grouped_kernel(const int* __restrict__ offs, int groups, int total_m, int N, int K,
                            const InT* __restrict__ A, long long lda, const InT* __restrict__ B, long long b_rs,
                            long long b_cs, long long b_gs, OutT* __restrict__ C, long long ldc, int axpby, float alpha,
                            float beta) {
  __shared__ int grp_end[kMaxGroups + 1];
  __shared__ int grp_blk[kMaxGroups + 1];
  __shared__ GenericTile As, Bs;
  group_table(offs, groups, total_m, 64, grp_end, grp_blk);
  const int q = blockIdx.x;
  if (q >= grp_blk[groups]) return;                  // the grid counts every group's blocks at their upper bound
  const int g = group_of(grp_blk, groups, q);
  const int m0 = (q - grp_blk[g]) * 64;
  for (int n0 = blockIdx.y * 64; n0 < N; n0 += gridDim.y * 64)
    generic_tile16(As, Bs, m0, n0, grp_end[g + 1] - grp_end[g], N, K, A + (long long)grp_end[g] * lda, lda, 1,
                   B + g * b_gs, b_rs, b_cs, C + (long long)grp_end[g] * ldc, ldc, axpby, alpha, beta);
}

// K-grouped (the weight gradient of a grouped layer): group g is K rows [end[g], end[g + 1]) of op(A) (M x total_k) and
// op(B) (total_k x N), element strides as gemm_generic_kernel's, and C_g = C + g * c_gs is a whole M x N matrix.  The
// groups run over blockIdx.z, gridDim.z at a time, and the row blocks over blockIdx.y, gridDim.y at a time.  An empty
// group stores what the 2-D call with k == 0 stores: round_out(beta * float(C)), or +0 without reading C when beta == 0.
template <typename InT, typename OutT>
__global__ void __launch_bounds__(256)
gemm_generic_kgrouped_kernel(const int* __restrict__ offs, int groups, int M, int N, int total_k,
                             const InT* __restrict__ A, long long a_rs, long long a_cs, const InT* __restrict__ B,
                             long long b_rs, long long b_cs, OutT* __restrict__ C, long long ldc, long long c_gs,
                             int axpby, float alpha, float beta) {
  __shared__ int grp_end[kMaxGroups + 1];
  __shared__ int grp_blk[kMaxGroups + 1];
  __shared__ GenericTile As, Bs;
  group_table(offs, groups, total_k, 64, grp_end, grp_blk);         // only the K ends are used
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int n0 = blockIdx.x * 64;
  for (int g = blockIdx.z; g < groups; g += gridDim.z) {
    const int k0 = grp_end[g], kg = grp_end[g + 1] - k0;
    OutT* Cg = C + g * c_gs;
    for (int m0 = blockIdx.y * 64; m0 < M; m0 += gridDim.y * 64) {
      if (kg > 0) {
        generic_tile16(As, Bs, m0, n0, M, N, kg, A + k0 * a_cs, a_rs, a_cs, B + k0 * b_rs, b_rs, b_cs, Cg, ldc, axpby,
                       alpha, beta);
        continue;
      }
      for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) {
          const int gm = m0 + ty + 16 * i, gn = n0 + tx + 16 * j;
          if (gm >= M || gn >= N) continue;
          OutT* e = Cg + (long long)gm * ldc + gn;
          store_out<float, OutT>(e, axpby && beta != 0.f ? beta * LoadAs<OutT>::ld(e) : 0.f);
        }
    }
  }
}

// The rows a grouped call writes, min(max(0, offs[0..groups)), total_m) = end[groups] of group_table, computed by
// every thread of the block.
__device__ __forceinline__ int grouped_rows(const int* __restrict__ offs, int groups, int total_m, int* s_max) {
  if (threadIdx.x == 0) *s_max = 0;
  __syncthreads();
  int v = 0;
  for (int i = threadIdx.x; i < groups; i += blockDim.x) v = max(v, offs[i]);
  atomicMax(s_max, v);
  __syncthreads();
  return min(*s_max, total_m);
}

// scale_inplace_kernel (s != 0) and fill_zero_kernel (s == 0) over rows [0, end[groups]): the k == 0 / alpha == 0
// pass of a grouped call.
template <typename T>
__global__ void scale_inplace_grouped_kernel(const int* __restrict__ offs, int groups, int total_m, int N,
                                             T* __restrict__ C, long long ldc, float s) {
  __shared__ int s_max;
  const int M = grouped_rows(offs, groups, total_m, &s_max);
  for (int r = blockIdx.y; r < M; r += gridDim.y)
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < N; c += gridDim.x * blockDim.x) {
      T* e = C + (long long)r * ldc + c;
      store_out<float, T>(e, s * LoadAs<T>::ld(e));
    }
}
template <typename T>
__global__ void fill_zero_grouped_kernel(const int* __restrict__ offs, int groups, int total_m, int N,
                                         T* __restrict__ C, long long ldc) {
  __shared__ int s_max;
  const int M = grouped_rows(offs, groups, total_m, &s_max);
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  for (int i = blockIdx.y; i < M; i += gridDim.y) C[(long long)i * ldc + j] = (T)0;
}

}  // namespace b200
