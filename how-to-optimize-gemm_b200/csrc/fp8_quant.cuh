// fp8_quant.cuh — blockwise FP8 quantisers: the producers of b200_gemm_fp8_blockwise's operands (DESIGN §4.7.6).
//
//   x (rows x cols, bf16 / fp16 / fp32, row-major, any pitch)  ->  q (FP8, rows x cols) + scales
//                                                                   [+ qt (FP8, cols x rows) + its scales]
// Recipes (BLK):
//   1    one scale per row and 128-column block (1 x 128: activations and gradients); with TRANS, qt holds x^T
//        quantised the same way, i.e. one scale per column of x and 128-row block (x's 128 x 1 blocks).
//   128  one scale per 128 x 128 block (weights); with TRANS, qt = q^T byte for byte and the scales are shared.
// The rule is the dynamic 1 x 128 epilogue's (fp8_q8_tile, gemm_tc.cuh): amax = max.NaN |x| over the block's elements
// inside the matrix, d = q8_block_scale(amax) (rn(amax / F), 1 when that is 0, NaN for a NaN or an inf), and
// c = cvt_fp8x2(rn(x / d)) (round to nearest even, finite values saturated to +-F, NaN kept).
//
// One CTA of 256 threads per 128 x 128 tile, persistent over (entry, tile row, tile column), tiles rastered along the
// columns of x.  A tile holds exactly one block of every recipe: one 1 x 128 block per row, one 128 x 1 block per
// column and one 128 x 128 block.  Each thread loads 16 bytes of x per pass (VEC elements of one row: LPR lanes per
// row), holds them as raw input bits, and takes its row's amax with shuffles inside the LPR lanes.  q is written from
// those registers.  With TRANS the tile is also staged in shared memory as raw input (rows padded by 16 bytes, so the
// 16-byte row stores and the 32-column reads are conflict-free); thread (half h, column j) then reduces 64 rows of
// column j, the two halves meet in shared memory, and it writes its 64 bytes of qt row j as 16-byte stores.
// A base, pitch or entry stride of x that is not 16-byte aligned takes element loads (vec = 0), and an output
// address that is not aligned takes byte stores, with the same bits.  All offsets are 64-bit.
#pragma once
#include "gemm_tc.cuh"

namespace b200 {

// Input element types: raw storage and the exact conversion to fp32 (-0, subnormals, inf and NaN kept).
struct qin_bf16 {
  using Raw = uint16_t;
  static __device__ __forceinline__ float f(uint16_t v) { return __uint_as_float((uint32_t)v << 16); }
};
// fp16: one cvt.f32.f16, exact
struct qin_f16 {
  using Raw = uint16_t;
  static __device__ __forceinline__ float f(uint16_t v) {
    float r;
    asm("cvt.f32.f16 %0, %1;" : "=f"(r) : "h"(v));
    return r;
  }
};
struct qin_f32 {
  using Raw = float;
  static __device__ __forceinline__ float f(float v) { return v; }
};

// One call: batch entries of a rows x cols matrix.  Element strides (x in input elements, q / qt in bytes, the scales
// in floats); st is null for the 128 x 128 recipe and qt null without the transposed output.
struct Fp8QuantArgs {
  const void* x; long long ldx, stride_x;
  uint8_t* q; long long ldq, stride_q;
  float* s; long long s_row, s_blk, s_entry;
  uint8_t* qt; long long ldqt, stride_qt;
  float* st; long long st_row, st_blk, st_entry;
  int rows, cols;
  int tiles_c;                    // ceil(cols / 128)
  long long tiles_entry, tiles;   // tiles of one entry, of the call
  int vec;                        // x's base, pitch and entry stride allow 16-byte loads
};

constexpr int kQuantThreads = 256;
// Shared-memory row pitch of the staged tile: 128 raw elements plus 16 bytes.
template <typename In>
__host__ __device__ constexpr int quant_pitch_bytes() { return 128 * (int)sizeof(typename In::Raw) + 16; }
template <typename In>
__host__ __device__ constexpr int quant_smem_bytes() { return 128 * quant_pitch_bytes<In>(); }

// n FP8 bytes of row pointer dst (n <= 16, values in w[], four per word): one store of 16 / 8 / 4 bytes where the
// address allows and all n are wanted, else byte stores of the first `valid`.
template <int N>
__device__ __forceinline__ void store_fp8_run(uint8_t* dst, const uint32_t (&w)[N / 4], int valid) {
  if (valid >= N && (reinterpret_cast<uintptr_t>(dst) & (N - 1)) == 0) {
    if constexpr (N == 16) *reinterpret_cast<uint4*>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
    else if constexpr (N == 8) *reinterpret_cast<uint2*>(dst) = make_uint2(w[0], w[1]);
    else *reinterpret_cast<uint32_t*>(dst) = w[0];
  } else {
#pragma unroll
    for (int i = 0; i < N; i++)
      if (i < valid) dst[i] = (uint8_t)(w[i / 4] >> (8 * (i % 4)));
  }
}

template <typename In, typename OutT, int BLK, bool TRANS>
__global__ void __launch_bounds__(kQuantThreads, 2) fp8_quant_kernel(const Fp8QuantArgs a) {
  using Raw = typename In::Raw;
  constexpr int VEC = 16 / (int)sizeof(Raw);          // elements per 16-byte load: 8 (16-bit) or 4 (fp32)
  constexpr int LPR = 128 / VEC;                      // lanes per tile row: 16 or 32
  constexpr int RPP = kQuantThreads / LPR;            // tile rows per pass: 16 or 8
  constexpr int PASSES = 128 / RPP;                   // 8 or 16
  constexpr int PITCH = quant_pitch_bytes<In>();
  extern __shared__ __align__(16) unsigned char quant_tile[];
  __shared__ float red[2][128];                       // column amax of each half (1 x 128), warp amax (128 x 128)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int c_off = (tid % LPR) * VEC, r_in = tid / LPR;

  for (long long t = blockIdx.x; t < a.tiles; t += gridDim.x) {
    const long long e = t / a.tiles_entry;
    const long long rem = t - e * a.tiles_entry;
    const int tr = (int)(rem / a.tiles_c), tc = (int)(rem - (long long)tr * a.tiles_c);
    const int r0 = 128 * tr, c0 = 128 * tc, col = c0 + c_off;
    const Raw* x = static_cast<const Raw*>(a.x) + e * a.stride_x;
    const bool whole = a.vec && col + VEC <= a.cols;

    // ---- load: PASSES x VEC raw elements, zero outside the matrix (|0| leaves every amax as it is)
    alignas(16) Raw v[PASSES][VEC];
#pragma unroll
    for (int p = 0; p < PASSES; p++) {
      const int row = r0 + p * RPP + r_in;
      const Raw* src = x + (long long)row * a.ldx + col;
      if (row < a.rows && whole) {
        *reinterpret_cast<uint4*>(v[p]) = __ldcs(reinterpret_cast<const uint4*>(src));
      } else {
#pragma unroll
        for (int i = 0; i < VEC; i++) v[p][i] = row < a.rows && col + i < a.cols ? src[i] : Raw(0);
      }
    }

    if constexpr (TRANS) {   // staged now, so that v is dead once q is written
#pragma unroll
      for (int p = 0; p < PASSES; p++)
        *reinterpret_cast<uint4*>(quant_tile + (p * RPP + r_in) * PITCH + c_off * (int)sizeof(Raw)) =
            *reinterpret_cast<const uint4*>(v[p]);
    }

    // ---- q from the registers, VEC bytes per row and pass, and its scales
    uint8_t* q = a.q + e * a.stride_q;
    auto store_q = [&](int p, float d) {
      const int row = r0 + p * RPP + r_in;
      uint32_t w[VEC / 4];
#pragma unroll
      for (int i = 0; i < VEC; i += 4) {
        const uint32_t lo = cvt_fp8x2<OutT>(__fdiv_rn(In::f(v[p][i]), d), __fdiv_rn(In::f(v[p][i + 1]), d));
        const uint32_t hi = cvt_fp8x2<OutT>(__fdiv_rn(In::f(v[p][i + 2]), d), __fdiv_rn(In::f(v[p][i + 3]), d));
        w[i / 4] = lo | (hi << 16);
      }
      if (row < a.rows && col < a.cols) store_fp8_run<VEC>(q + (long long)row * a.ldq + col, w, a.cols - col);
    };
    float d_tile = 0.f;      // 128 x 128: the tile's scale
    if constexpr (BLK == 1) {
#pragma unroll
      for (int p = 0; p < PASSES; p++) {
        float m = 0.f;
#pragma unroll
        for (int i = 0; i < VEC; i++) m = fmax_nan(m, fabsf(In::f(v[p][i])));
#pragma unroll
        for (int o = LPR / 2; o > 0; o >>= 1) m = fmax_nan(m, __shfl_xor_sync(0xffffffffu, m, o));
        const float d = q8_block_scale<OutT>(m);
        const int row = r0 + p * RPP + r_in;
        if (tid % LPR == 0 && row < a.rows) a.s[e * a.s_entry + row * a.s_row + tc * a.s_blk] = d;
        store_q(p, d);
      }
    } else {
      float m = 0.f;
#pragma unroll
      for (int p = 0; p < PASSES; p++)
#pragma unroll
        for (int i = 0; i < VEC; i++) m = fmax_nan(m, fabsf(In::f(v[p][i])));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmax_nan(m, __shfl_xor_sync(0xffffffffu, m, o));
      if (lane == 0) red[0][warp] = m;
      __syncthreads();
      m = red[0][0];
#pragma unroll
      for (int w = 1; w < kQuantThreads / 32; w++) m = fmax_nan(m, red[0][w]);
      d_tile = q8_block_scale<OutT>(m);
      if (tid == 0) a.s[e * a.s_entry + tr * a.s_row + tc * a.s_blk] = d_tile;
#pragma unroll
      for (int p = 0; p < PASSES; p++) store_q(p, d_tile);
    }

    if constexpr (TRANS) {
      // ---- qt: one thread per (half, column) reads 64 rows of the column from the staged tile
      __syncthreads();
      const int cl = (warp & 3) * 32 + lane, h = warp >> 2, j = c0 + cl;
      const unsigned char* colp = quant_tile + (h * 64) * PITCH + cl * (int)sizeof(Raw);
      auto val = [&](int r) { return In::f(*reinterpret_cast<const Raw*>(colp + r * PITCH)); };
      float dt;
      if constexpr (BLK == 1) {
        float m = 0.f;
#pragma unroll 16
        for (int r = 0; r < 64; r++) m = fmax_nan(m, fabsf(val(r)));
        red[h][cl] = m;
        __syncthreads();
        dt = q8_block_scale<OutT>(fmax_nan(red[0][cl], red[1][cl]));
        if (h == 0 && j < a.cols) a.st[e * a.st_entry + (long long)j * a.st_row + tr * a.st_blk] = dt;
      } else {
        dt = d_tile;
      }
      if (j < a.cols) {
        const int i0 = r0 + h * 64;
        uint8_t* dst = a.qt + e * a.stride_qt + (long long)j * a.ldqt + i0;
#pragma unroll
        for (int c = 0; c < 4; c++) {
          uint32_t w[4];
#pragma unroll
          for (int i = 0; i < 16; i += 4) {
            const int r = 16 * c + i;
            const uint32_t lo = cvt_fp8x2<OutT>(__fdiv_rn(val(r), dt), __fdiv_rn(val(r + 1), dt));
            const uint32_t hi = cvt_fp8x2<OutT>(__fdiv_rn(val(r + 2), dt), __fdiv_rn(val(r + 3), dt));
            w[i / 4] = lo | (hi << 16);
          }
          if (i0 + 16 * c < a.rows) store_fp8_run<16>(dst + 16 * c, w, a.rows - (i0 + 16 * c));
        }
      }
    }
    __syncthreads();   // the next tile reuses red[] and the staged tile
  }
}

}  // namespace b200
