// gemm_mxf4.cuh — the 4-bit path (SURVEY §8 f-4): block-scaled MXFP4 operands.
//
// The reference lists a `cuda-int4` back-end and ships only the word "WIP" (cuda-int4/README.md:1,
// README.md:13-15,118-120).  The 4-bit operand type here is OCP MXFP4: E2M1 elements
// (+-{0, .5, 1, 1.5, 2, 3, 4, 6}) with one shared UE8M0 scale (a power of two) per 32 consecutive K elements.
// This file holds
//   * the quantisers: fp32 rows -> packed E2M1 + scales (A as stored), and the transposing variant for a
//     row-major B (4-bit operands are stored K-major — the one place where the reorder_b / trans_w role of
//     aarch64-int8/MMult_4x8_21.c:45-71 does come back as a real pass);
//   * the expansion of quantised operands to bf16 for the GEMM (see "the GEMM on sm_90" below).
//
// Layouts in HBM
//   elements  rows x (k/2) bytes, two E2M1 per byte (element 2i in the low nibble), K contiguous;
//   scales    512-byte atoms [rows/128][k/128]: byte (r % 32) * 16 + ((r / 32) % 4) * 4 + (kblock % 4) of the
//             atom holds the UE8M0 scale of row r, K-block kblock.
#pragma once
#include <cuda_bf16.h>

#include "ptx.cuh"

namespace b200 {

// ---- E2M1 / UE8M0 arithmetic (device side; oracle/oracle.c holds the host restatement) ----------------
// Round-to-nearest-even of |v| <= 6 onto {0, .5, 1, 1.5, 2, 3, 4, 6}; larger magnitudes saturate at 6.
__device__ __forceinline__ uint32_t e2m1_encode(float v) {
  const uint32_t sign = (__float_as_uint(v) >> 31) << 3;
  const float a = fabsf(v);
  // midpoints of the grid; a tie goes to the neighbour with an even (zero) mantissa bit: 0, 1, 2, 4
  const uint32_t code = a <= 0.25f ? 0u : a < 0.75f ? 1u : a <= 1.25f ? 2u : a < 1.75f ? 3u
                      : a <= 2.5f ? 4u : a < 3.5f ? 5u : a <= 5.0f ? 6u : 7u;
  return (a != a) ? 0u : (sign | code);            // E2M1 has no NaN: a NaN element becomes +0 (its block scale is NaN)
}
// Shared scale of a 32-element block (OCP MX v1.0 §6.3): 2^(floor(log2(max|x|)) - 2), 2 = emax of E2M1.
// Returns the biased UE8M0 exponent; an all-zero (or denormal) block takes the smallest scale.
__device__ __forceinline__ uint32_t ue8m0_from_max(float mx) {
  const int ef = (int)((__float_as_uint(mx) >> 23) & 0xFF);    // biased exponent of max = floor(log2) + 127
  if (ef == 255) return 255u;                                    // inf / NaN block -> NaN scale
  const int e = ef - 2;
  return (uint32_t)(e < 0 ? 0 : e);
}
__device__ __forceinline__ float ue8m0_inv(uint32_t e) {         // 2^-(e - 127), clamped to normal floats
  int x = 254 - (int)e;
  x = x < 1 ? 1 : (x > 254 ? 254 : x);
  return __uint_as_float((uint32_t)x << 23);
}
__device__ __forceinline__ float exp2i_small(int e) { return __uint_as_float((uint32_t)(127 + e) << 23); }
__host__ __device__ __forceinline__ size_t mxf4_sf_offset(int r, int kblock, int katoms) {
  return ((size_t)(r >> 7) * katoms + (kblock >> 2)) * 512 + (size_t)(r & 31) * 16 + ((r >> 5) & 3) * 4 + (kblock & 3);
}

// One warp quantises one 32-element block per lane-group: thread = one block of 32 consecutive K elements
// of one row (rows x cols fp32, pitch ld; cols padded with zeros to a multiple of 128 in the outputs).
__global__ void __launch_bounds__(256) mxf4_quantize_rows_kernel(const float* __restrict__ src, long long ld, int rows,
                                                                 int cols, uint8_t* __restrict__ q, int kpad,
                                                                 uint8_t* __restrict__ sf, int rows_pad) {
  const int kblocks = kpad >> 5, katoms = kpad >> 7;
  const long long total = (long long)rows_pad * kblocks;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / kblocks), kb = (int)(i - (long long)r * kblocks);
    float x[32];
    float mx = 0.f;
#pragma unroll
    for (int e = 0; e < 32; e++) {
      const int c = kb * 32 + e;
      x[e] = (r < rows && c < cols) ? src[(long long)r * ld + c] : 0.f;
      mx = fmaxf(mx, fabsf(x[e]));
    }
    const uint32_t se = ue8m0_from_max(mx);
    const float inv = ue8m0_inv(se);
    sf[mxf4_sf_offset(r, kb, katoms)] = (uint8_t)se;
    if (r < rows) {
      uint32_t w[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        uint32_t v = 0;
#pragma unroll
        for (int e = 0; e < 8; e++) v |= e2m1_encode(x[j * 8 + e] * inv) << (4 * e);
        w[j] = v;
      }
      *reinterpret_cast<uint4*>(q + (long long)r * (kpad >> 1) + kb * 16) = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
}

// Transposing quantiser for a row-major B (k x n): block = 32 k-rows x 256 n-columns through shared memory,
// then thread = one column: its 32 values along K are one scale block.  Output rows are the COLUMNS of B.  A block
// takes the K-blocks blockIdx.y, + gridDim.y, ... (gridDim.y is capped at 65535: one unless kpad > 2097120).
__global__ void __launch_bounds__(256) mxf4_quantize_cols_t_kernel(const float* __restrict__ src, long long ld, int krows,
                                                                   int ncols, uint8_t* __restrict__ q, int kpad,
                                                                   uint8_t* __restrict__ sf, int n_pad) {
  __shared__ float tile[32][257];
  const int n0 = blockIdx.x * 256, katoms = kpad >> 7, kblocks = kpad >> 5;
  const int n = n0 + threadIdx.x;
  for (int kb = blockIdx.y; kb < kblocks; kb += gridDim.y) {
    if (kb != (int)blockIdx.y) __syncthreads();        // the previous K-block's reads of `tile` are done
    for (int rr = threadIdx.x >> 6; rr < 32; rr += 4) {
      const int kr = kb * 32 + rr;
#pragma unroll
      for (int cc = 0; cc < 4; cc++) {
        const int c = (threadIdx.x & 63) + cc * 64;
        tile[rr][c] = (kr < krows && n0 + c < ncols) ? src[(long long)kr * ld + n0 + c] : 0.f;
      }
    }
    __syncthreads();
    if (n >= n_pad) continue;
    float mx = 0.f;
#pragma unroll
    for (int e = 0; e < 32; e++) mx = fmaxf(mx, fabsf(tile[e][threadIdx.x]));
    const uint32_t se = ue8m0_from_max(mx);
    const float inv = ue8m0_inv(se);
    sf[mxf4_sf_offset(n, kb, katoms)] = (uint8_t)se;
    if (n < ncols) {
      uint32_t w[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        uint32_t v = 0;
#pragma unroll
        for (int e = 0; e < 8; e++) v |= e2m1_encode(tile[j * 8 + e][threadIdx.x] * inv) << (4 * e);
        w[j] = v;
      }
      *reinterpret_cast<uint4*>(q + (long long)n * (kpad >> 1) + kb * 16) = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
}

// ---- the GEMM on sm_90 -------------------------------------------------------------------------------------
// Hopper's tensor cores take no 4-bit operand.  An E2M1 element times its UE8M0 block scale is exactly a bf16
// (one mantissa bit; the scale only moves the exponent), so both operands are expanded to bf16 — A as m x kpad
// row-major, B^T back to row-major kpad x n — and multiplied by the bf16 wgmma kernel (gemm_tc.cuh) with fp32
// accumulation: every product is exact, as in a block-scaled MMA.
__device__ __forceinline__ float e2m1_decode(uint32_t c) {
  const uint32_t m = c & 7u;
  const float mag = m < 2 ? 0.5f * (float)m : (float)(2 + (m & 1)) * exp2i_small((int)(m >> 1) - 2);
  return (c & 8u) ? -mag : mag;
}
__device__ __forceinline__ float ue8m0_value(uint32_t e) {       // 2^(e - 127); 255 is NaN
  if (e == 255u) return __uint_as_float(0x7FC00000u);
  return e == 0u ? __uint_as_float(0x00400000u) : __uint_as_float(e << 23);
}
// 32 consecutive K elements of one row -> bf16 (RNE of an exact value: no rounding happens)
__device__ __forceinline__ void mxf4_expand32(const uint8_t* q, uint32_t se, float (&x)[32]) {
  const uint4 v = *reinterpret_cast<const uint4*>(q);
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  const float s = ue8m0_value(se);
#pragma unroll
  for (int e = 0; e < 32; e++) x[e] = e2m1_decode((w[e >> 3] >> (4 * (e & 7))) & 15u) * s;
}

// A: rows x kpad/2 bytes -> rows x kpad bf16 (pitch kpad).  Thread = one 32-element block.
__global__ void __launch_bounds__(256) mxf4_expand_rows_kernel(const uint8_t* __restrict__ q, const uint8_t* __restrict__ sf,
                                                               int rows, int kpad, uint16_t* __restrict__ dst) {
  griddep_launch();
  griddep_wait();
  const int kblocks = kpad >> 5, katoms = kpad >> 7;
  const long long total = (long long)rows * kblocks;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / kblocks), kb = (int)(i - (long long)r * kblocks);
    float x[32];
    mxf4_expand32(q + (long long)r * (kpad >> 1) + kb * 16, sf[mxf4_sf_offset(r, kb, katoms)], x);
    uint4* d = reinterpret_cast<uint4*>(dst + (long long)r * kpad + kb * 32);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      uint32_t w[4];
#pragma unroll
      for (int e = 0; e < 4; e++) {
        uint32_t r2;
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r2) : "f"(x[8 * j + 2 * e + 1]), "f"(x[8 * j + 2 * e]));
        w[e] = r2;
      }
      d[j] = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
}

// B^T: n x kpad/2 bytes -> row-major kpad x n bf16 (pitch dld).  Thread = one column n and the 32-row K-blocks
// blockIdx.y, + gridDim.y, ... (gridDim.y is capped at 65535: one unless kpad > 2097120); neighbouring threads write
// neighbouring columns.
__global__ void __launch_bounds__(256) mxf4_expand_cols_t_kernel(const uint8_t* __restrict__ q, const uint8_t* __restrict__ sf,
                                                                 int n, int kpad, uint16_t* __restrict__ dst, long long dld) {
  griddep_launch();
  griddep_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x, katoms = kpad >> 7, kblocks = kpad >> 5;
  if (c >= n) return;
  for (int kb = blockIdx.y; kb < kblocks; kb += gridDim.y) {
    float x[32];
    mxf4_expand32(q + (long long)c * (kpad >> 1) + kb * 16, sf[mxf4_sf_offset(c, kb, katoms)], x);
#pragma unroll
    for (int e = 0; e < 32; e++) dst[(long long)(kb * 32 + e) * dld + c] = __bfloat16_as_ushort(__float2bfloat16_rn(x[e]));
  }
}

}  // namespace b200
