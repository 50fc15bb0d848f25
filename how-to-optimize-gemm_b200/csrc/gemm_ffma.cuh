// gemm_ffma.cuh — the strict-fp32 path: CUDA-core SGEMM for sm_90a, fed by TMA, FFMA math.
//
// Arithmetic contract (what makes this the drop-in for cuda/MMult_cuda_12.cu:200-206 and bit-exact
// against the reference's naive oracle as its own makefile builds it, aarch64/REF_MMult.cpp:24 with
// GCC's fused multiply-add): every C(i,j) is ONE accumulator chain
//     c = 0 (or C(i,j));  for p = 0..k-1 (ascending):  c = fma(A(i,p), B(p,j), c)
// no split-K, no reassociation.
//
// Structure: 128x128 CTA tile, 256 threads (8 warps laid out 4(ty) x 8(tx) lanes), 8x8 outputs per
// thread as rows ty+16*i, column groups tx*4+64*j.  The reference's gmem->reg->smem double buffer
// (cuda/MMult_cuda_12.cu:113-198) becomes a 3-deep TMA ring guarded by mbarriers: no LDG/STS issue
// slots are spent on staging.  A lands K-contiguous with SWIZZLE_128B so four consecutive rows read
// by a warp hit distinct banks; B lands N-contiguous (512-byte rows).
//
// Math: the accumulators are kept as float2 pairs (two adjacent columns); each pair is updated by two
// IEEE fmas (ffma2 below), so every element is one fused multiply-add chain.
//
// Wave quantisation: 2 CTAs/SM x 132 SMs = 264 slots.  Tiles beyond the last full round are issued as
// two HALF tiles (rows ty+16*i for i in [0,4) or [4,8)) when that fills the machine better — each
// half is still a complete sequential-k chain per element, so the contract above is untouched.
#pragma once
#include "ptx.cuh"

namespace b200 {

__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}

__device__ __forceinline__ float2 lds64(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}

// d = a * b + c on both halves of a float2 pair, each a single-rounding fma
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

struct FfmaParams {
  float* C;
  long long ldc;
  int M, N, K;
  int vec_ok;
  int accumulate;   // 1: accumulator chains start from C(i,j) (C += A*B), 0: from zero (C = A*B)
  int tiles_m, tiles_n, group_m;
  int full_tiles;   // CTAs [0, full_tiles) own whole tiles; later CTAs own half tiles, two per tile
  // General epilogue C = alpha * (A*B) + beta * C (b200_gemm_f32_ex), axpby == 1 only; the chains then start
  // from zero and C is read only when beta != 0.
  int axpby;
  float alpha, beta;
};

// Four adjacent outputs ev (columns gn..gn+3 of one row, dst = &C(row, gn)) through the general epilogue, with
// the arithmetic of the tensor-core epilogue: alpha * v rounded, then fma(beta, C, .).
__device__ __forceinline__ void ffma_axpby4(const FfmaParams& p, const float* dst, int gn, bool vec, float (&ev)[4]) {
#pragma unroll
  for (int e = 0; e < 4; e++) ev[e] *= p.alpha;
  if (p.beta == 0.f) return;
  if (vec) {
    const float4 o = *reinterpret_cast<const float4*>(dst);
    ev[0] = fmaf(p.beta, o.x, ev[0]); ev[1] = fmaf(p.beta, o.y, ev[1]);
    ev[2] = fmaf(p.beta, o.z, ev[2]); ev[3] = fmaf(p.beta, o.w, ev[3]);
  } else {
#pragma unroll
    for (int e = 0; e < 4; e++)
      if (gn + e < p.N) ev[e] = fmaf(p.beta, dst[e], ev[e]);
  }
}

struct FfmaCfg {
  static constexpr int BM = 128, BN = 128, BK = 32, STAGES = 3;
  static constexpr int A_STAGE = BM * BK * 4;     // 16 KB, 128 rows x 128 B (swizzled)
  static constexpr int B_STAGE = BK * BN * 4;     // 16 KB, 32 rows x 512 B
  static constexpr int STAGE_BYTES = A_STAGE + B_STAGE;
  static constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + 2 * STAGES * 8;
  static constexpr int THREADS = 256;
};

// Main loop + epilogue for NI row-groups per thread starting at row-group i0 (NI = 8: whole tile).
template <int NI>
__device__ __forceinline__ void ffma_tile(const CUtensorMap& tmA, const CUtensorMap& tmB, const FfmaParams& p,
                                          int m0, int n0, int i0, uint32_t sA, uint32_t sB,
                                          uint32_t bar_full, uint32_t bar_empty) {
  using Cfg = FfmaCfg;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ty = (warp >> 1) * 4 + (lane >> 3);   // 0..15
  const int tx = (warp & 1) * 8 + (lane & 7);     // 0..15
  const int num_kb = (p.K + Cfg::BK - 1) / Cfg::BK;

  auto issue = [&](int kb) {                        // thread 0 only
    const int s = kb % Cfg::STAGES;
    const uint32_t full = bar_full + 8 * s;
    mbar_arrive_expect_tx(full, Cfg::STAGE_BYTES);
    tma_load_2d(sA + s * Cfg::A_STAGE, &tmA, full, kb * Cfg::BK, m0);
    tma_load_2d(sB + s * Cfg::B_STAGE, &tmB, full, n0, kb * Cfg::BK);
  };
  if (threadIdx.x == 0) {
    for (int kb = 0; kb < Cfg::STAGES - 1 && kb < num_kb; kb++) issue(kb);
  }

  float2 acc[NI][4];
#pragma unroll
  for (int i = 0; i < NI; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = make_float2(0.0f, 0.0f);
  if (p.accumulate) {
#pragma unroll
    for (int i = 0; i < NI; i++)
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const int gm = m0 + ty + 16 * (i0 + i), gn = n0 + tx * 4 + 64 * (j >> 2) + (j & 3);
        if (gm < p.M && gn < p.N) {
          const float v = p.C[(long long)gm * p.ldc + gn];
          if (j & 1) acc[i][j >> 1].y = v; else acc[i][j >> 1].x = v;
        }
      }
  }

  // 32-bit shared-window addresses (cf. smem_u32addr / lds128 in cuda/MMult_cuda_10.cu:31-48): one
  // register per operand stream, immediates for everything else, so nothing is re-derived from
  // threadIdx inside the loop.  A rows ty+16*i all share (row & 7) == (ty & 7).
  const uint32_t a_thr = sA + (ty + 16 * i0) * 128;   // + stage + i*2048 + ((kc << 4) ^ a_swz16)
  const uint32_t a_swz16 = (ty & 7) << 4;
  const uint32_t b_thr = sB + tx * 16;                // + stage + k*512 (+256)

  for (int kb = 0; kb < num_kb; kb++) {
    const int s = kb % Cfg::STAGES;
    const uint32_t use = kb / Cfg::STAGES;
    if (threadIdx.x == 0) {
      const int nk = kb + Cfg::STAGES - 1;           // refill the slot consumed in iteration kb-1
      if (nk < num_kb) {
        if (kb >= 1) mbar_wait(bar_empty + 8 * (nk % Cfg::STAGES), ((nk / Cfg::STAGES) - 1) & 1);
        issue(nk);
      }
    }
    mbar_wait(bar_full + 8 * s, use & 1);
    const uint32_t a_st = a_thr + s * Cfg::A_STAGE;
    const uint32_t b_st = b_thr + s * Cfg::B_STAGE;
    // Fully unrolled over the stage (8 x [8 LDS.128 of A + 4 x (2 LDS.128 of B + 64 FFMA)]).
#pragma unroll
    for (int kc = 0; kc < Cfg::BK / 4; kc++) {
      float4 a4[NI];
#pragma unroll
      for (int i = 0; i < NI; i++)
        a4[i] = lds128(a_st + (((uint32_t)kc << 4) ^ a_swz16) + i * (16 * 128));
#pragma unroll
      for (int kk = 0; kk < 4; kk++) {
        const float4 b0 = lds128(b_st + (kc * 4 + kk) * 512);
        const float4 b1 = lds128(b_st + (kc * 4 + kk) * 512 + 256);
        const float2 bv[4] = {make_float2(b0.x, b0.y), make_float2(b0.z, b0.w),
                              make_float2(b1.x, b1.y), make_float2(b1.z, b1.w)};
#pragma unroll
        for (int i = 0; i < NI; i++) {
          const float av = kk == 0 ? a4[i].x : kk == 1 ? a4[i].y : kk == 2 ? a4[i].z : a4[i].w;
          const float2 aa = make_float2(av, av);
#pragma unroll
          for (int j = 0; j < 4; j++) acc[i][j] = ffma2(aa, bv[j], acc[i][j]);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * s);
  }

  // epilogue: 16-byte stores; for fixed (i, j) a warp writes 4 rows x 128 contiguous bytes
#pragma unroll
  for (int i = 0; i < NI; i++) {
    const int gm = m0 + ty + 16 * (i0 + i);
    if (gm >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 2; j++) {
      const int gn = n0 + tx * 4 + 64 * j;
      float* dst = p.C + (long long)gm * p.ldc + gn;
      const bool vec = p.vec_ok && gn + 4 <= p.N;
      float ev[4] = {acc[i][2 * j].x, acc[i][2 * j].y, acc[i][2 * j + 1].x, acc[i][2 * j + 1].y};
      if (p.axpby) ffma_axpby4(p, dst, gn, vec, ev);
      if (vec) {
        *reinterpret_cast<float4*>(dst) = make_float4(ev[0], ev[1], ev[2], ev[3]);
      } else {
#pragma unroll
        for (int e = 0; e < 4; e++)
          if (gn + e < p.N) dst[e] = ev[e];
      }
    }
  }
}

__global__ void __launch_bounds__(256, 2)
gemm_ffma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const FfmaParams p) {
  using Cfg = FfmaCfg;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sA = smem_base;
  const uint32_t sB = sA + Cfg::STAGES * Cfg::A_STAGE;
  const uint32_t bar_full = sB + Cfg::STAGES * Cfg::B_STAGE;
  const uint32_t bar_empty = bar_full + 8 * Cfg::STAGES;

  // work decode: whole tiles first (m-fastest inside groups of group_m row-blocks, for L2 reuse of
  // the B column panel), then the half tiles of the last partial round
  const int b = blockIdx.x;
  int tile = b, i0 = 0;
  const bool half = b >= p.full_tiles;
  if (half) {
    const int r = b - p.full_tiles;
    tile = p.full_tiles + (r >> 1);
    i0 = (r & 1) * 4;
  }
  const int per_group = p.group_m * p.tiles_n;
  const int g = tile / per_group;
  const int first_m = g * p.group_m;
  const int rows = min(p.group_m, p.tiles_m - first_m);
  const int rr = tile - g * per_group;
  const int m0 = (first_m + rr % rows) * Cfg::BM, n0 = (rr / rows) * Cfg::BN;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < Cfg::STAGES; i++) {
      mbar_init(bar_full + 8 * i, 1);
      mbar_init(bar_empty + 8 * i, 8);             // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (!half) ffma_tile<8>(tmA, tmB, p, m0, n0, 0, sA, sB, bar_full, bar_empty);
  else       ffma_tile<4>(tmA, tmB, p, m0, n0, i0, sA, sB, bar_full, bar_empty);
}


// ---------------------------------------------------------------------------------------------------
// "Fat-thread" variant: 128 x 256 CTA tile, 256 threads, 8 x 16 outputs per thread (128 accumulators,
// 1 CTA per SM, up to 255 registers).  Same arithmetic contract.  The larger register budget allows
// what the 128-register 8x8 kernel cannot: both operand streams are fetched one step ahead (A for the
// next 4 k-steps, B for the next k-step) while the current 128 FFMA issue, so no shared-memory latency
// is exposed at k-chunk boundaries, and each k-step needs 6 LDS.128 per 128 FFMA instead of 4 per 64.
struct FfmaFatCfg {
  static constexpr int BM = 128, BN = 256, BK = 32, STAGES = 3;
  static constexpr int A_STAGE = BM * BK * 4;     // 16 KB, swizzled 128 B rows
  static constexpr int B_STAGE = BK * BN * 4;     // 32 KB, 32 rows x 1024 B
  static constexpr int STAGE_BYTES = A_STAGE + B_STAGE;
  static constexpr int SMEM_BYTES = 1024 + STAGES * STAGE_BYTES + 2 * STAGES * 8;
  static constexpr int THREADS = 256;
};

template <int NI>
__device__ __forceinline__ void ffma_fat_tile(const CUtensorMap& tmA, const CUtensorMap& tmB, const FfmaParams& p,
                                              int m0, int n0, int i0, uint32_t sA, uint32_t sB,
                                              uint32_t bar_full, uint32_t bar_empty) {
  using Cfg = FfmaFatCfg;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ty = (warp >> 1) * 4 + (lane >> 3);   // 0..15 : rows ty + 16*i
  const int tx = (warp & 1) * 8 + (lane & 7);     // 0..15 : columns tx*4 + 64*j, j = 0..3
  const int num_kb = (p.K + Cfg::BK - 1) / Cfg::BK;

  auto issue = [&](int kb) {
    const int s = kb % Cfg::STAGES;
    const uint32_t full = bar_full + 8 * s;
    mbar_arrive_expect_tx(full, Cfg::STAGE_BYTES);
    tma_load_2d(sA + s * Cfg::A_STAGE, &tmA, full, kb * Cfg::BK, m0);
    tma_load_2d(sB + s * Cfg::B_STAGE, &tmB, full, n0, kb * Cfg::BK);
  };
  if (threadIdx.x == 0) {
    for (int kb = 0; kb < Cfg::STAGES - 1 && kb < num_kb; kb++) issue(kb);
  }

  float2 acc[NI][8];
#pragma unroll
  for (int i = 0; i < NI; i++)
#pragma unroll
    for (int j = 0; j < 8; j++) acc[i][j] = make_float2(0.0f, 0.0f);
  if (p.accumulate) {
#pragma unroll
    for (int i = 0; i < NI; i++)
#pragma unroll
      for (int j = 0; j < 16; j++) {
        const int gm = m0 + ty + 16 * (i0 + i), gn = n0 + tx * 4 + 64 * (j >> 2) + (j & 3);
        if (gm < p.M && gn < p.N) {
          const float v = p.C[(long long)gm * p.ldc + gn];
          if (j & 1) acc[i][j >> 1].y = v; else acc[i][j >> 1].x = v;
        }
      }
  }
  const uint32_t a_thr = sA + (ty + 16 * i0) * 128;
  const uint32_t a_swz16 = (ty & 7) << 4;
  const uint32_t b_thr = sB + tx * 16;

  for (int kb = 0; kb < num_kb; kb++) {
    const int s = kb % Cfg::STAGES;
    const uint32_t use = kb / Cfg::STAGES;
    if (threadIdx.x == 0) {
      const int nk = kb + Cfg::STAGES - 1;
      if (nk < num_kb) {
        if (kb >= 1) mbar_wait(bar_empty + 8 * (nk % Cfg::STAGES), ((nk / Cfg::STAGES) - 1) & 1);
        issue(nk);
      }
    }
    mbar_wait(bar_full + 8 * s, use & 1);
    const uint32_t a_st = a_thr + s * Cfg::A_STAGE;
    const uint32_t b_st = b_thr + s * Cfg::B_STAGE;
    float4 a4[2][NI];
    float4 bq[2][4];
#pragma unroll
    for (int i = 0; i < NI; i++) a4[0][i] = lds128(a_st + a_swz16 + i * (16 * 128));
#pragma unroll
    for (int j = 0; j < 4; j++) bq[0][j] = lds128(b_st + j * 256);
#pragma unroll
    for (int kc = 0; kc < Cfg::BK / 4; kc++) {
      const int ac = kc & 1;
      if (kc + 1 < Cfg::BK / 4) {
#pragma unroll
        for (int i = 0; i < NI; i++)
          a4[ac ^ 1][i] = lds128(a_st + (((uint32_t)(kc + 1) << 4) ^ a_swz16) + i * (16 * 128));
      }
#pragma unroll
      for (int kk = 0; kk < 4; kk++) {
        const int k = kc * 4 + kk;
        if (k + 1 < Cfg::BK) {
#pragma unroll
          for (int j = 0; j < 4; j++) bq[(k + 1) & 1][j] = lds128(b_st + (k + 1) * 1024 + j * 256);
        }
        float2 bv[8];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          bv[2 * j] = make_float2(bq[k & 1][j].x, bq[k & 1][j].y);
          bv[2 * j + 1] = make_float2(bq[k & 1][j].z, bq[k & 1][j].w);
        }
#pragma unroll
        for (int i = 0; i < NI; i++) {
          const float av = kk == 0 ? a4[ac][i].x : kk == 1 ? a4[ac][i].y : kk == 2 ? a4[ac][i].z : a4[ac][i].w;
          const float2 aa = make_float2(av, av);
#pragma unroll
          for (int j = 0; j < 8; j++) acc[i][j] = ffma2(aa, bv[j], acc[i][j]);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty + 8 * s);
  }

#pragma unroll
  for (int i = 0; i < NI; i++) {
    const int gm = m0 + ty + 16 * (i0 + i);
    if (gm >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int gn = n0 + tx * 4 + 64 * j;
      float* dst = p.C + (long long)gm * p.ldc + gn;
      const bool vec = p.vec_ok && gn + 4 <= p.N;
      float ev[4] = {acc[i][2 * j].x, acc[i][2 * j].y, acc[i][2 * j + 1].x, acc[i][2 * j + 1].y};
      if (p.axpby) ffma_axpby4(p, dst, gn, vec, ev);
      if (vec) {
        *reinterpret_cast<float4*>(dst) = make_float4(ev[0], ev[1], ev[2], ev[3]);
      } else {
#pragma unroll
        for (int e = 0; e < 4; e++)
          if (gn + e < p.N) dst[e] = ev[e];
      }
    }
  }
}

__global__ void __launch_bounds__(256, 1)
gemm_ffma_fat_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const FfmaParams p) {
  using Cfg = FfmaFatCfg;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sA = smem_base;
  const uint32_t sB = sA + Cfg::STAGES * Cfg::A_STAGE;
  const uint32_t bar_full = sB + Cfg::STAGES * Cfg::B_STAGE;
  const uint32_t bar_empty = bar_full + 8 * Cfg::STAGES;
  const int b = blockIdx.x;
  int tile = b, i0 = 0;
  const bool half = b >= p.full_tiles;
  if (half) {
    const int r = b - p.full_tiles;
    tile = p.full_tiles + (r >> 1);
    i0 = (r & 1) * 4;
  }
  const int per_group = p.group_m * p.tiles_n;
  const int g = tile / per_group;
  const int first_m = g * p.group_m;
  const int rows = min(p.group_m, p.tiles_m - first_m);
  const int rr = tile - g * per_group;
  const int m0 = (first_m + rr % rows) * Cfg::BM, n0 = (rr / rows) * Cfg::BN;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < Cfg::STAGES; i++) {
      mbar_init(bar_full + 8 * i, 1);
      mbar_init(bar_empty + 8 * i, 8);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (!half) ffma_fat_tile<8>(tmA, tmB, p, m0, n0, 0, sA, sB, bar_full, bar_empty);
  else       ffma_fat_tile<4>(tmA, tmB, p, m0, n0, i0, sA, sB, bar_full, bar_empty);
}

}  // namespace b200
