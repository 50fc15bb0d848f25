// gemm_tc.cuh — the tensor-core path: persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   C[m x n] = op(A) * op(B),  C row-major; each operand stored row-major as given (N) or as its transpose (T).
//   Operand kinds: bf16 (KIND_F16), fp16 (KIND_FP16), tf32, int8; C fp32 / int32, bf16, fp16 or requantised int8.
//
// Mapping of the reference's roles (SURVEY §8a) onto Hopper:
//   packA / packB  (aarch64/MMult_4x4_21.cpp:459-572; the gmem->smem staging of
//                   cuda/MMult_cuda_12.cu:113-198)      -> TMA bulk-tensor copies with hardware swizzle
//                                                          into a STAGES-deep shared-memory ring
//   4x4 / 8x12 register micro-kernel (kernel_8x12,
//                   cuda/MMult_cuda_12.cu:200-206)      -> two consumer warpgroups, each issuing
//                                                          wgmma 64 x BN x K into register accumulators
//   stg128 epilogue (cuda/MMult_cuda_12.cu:210-222)     -> stores straight from the accumulator registers
//
// Operand layouts in shared memory (template parameters AL / BL of the kernel, LAYOUT_K or LAYOUT_MN):
//   K-major:  rows of one operand's M (or N) index, BK elements of K per 128- or 64-byte swizzled row.  Row-major
//             A (m x k) and B^T (n x k) are K-major as stored.
//   MN-major: [BK k-rows x 128 B] column blocks of a k x m or k x n row-major matrix, SWIZZLE_128B, 8 k-rows per
//             1 KB atom; wgmma transposes them on the fly.  Row-major B (k x n) and A^T (k x m) are MN-major as
//             stored.  16-bit kinds only: the tile of A^T is the tile of row-major B, one 64-column box per consumer.
// tf32 and int8: wgmma takes only K-major operands for 32- and 8-bit types, so a row-major B or a transposed A
// is first transposed by transpose_kernel (the job of reorder_b / trans_w in aarch64-int8/MMult_4x8_21.c:45-71).
//
// Split-precision fp32 (B200_F32_BF16X3 / _BF16X2 / _F16X2): A and B arrive as NPA / NPB stacked 16-bit
// "planes" (a = a1 + a2 + a3, produced by split_planes_kernel); each k-block stage holds every plane once
// and the consumers issue the listed plane products into the SAME fp32 accumulator, smallest terms first.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread issues; the group gives its registers
// to the consumers), warpgroups 1 and 2 = consumers of rows [0, 64) and [64, 128) of the tile: each issues
// its wgmma chain and writes its own rows of C.  The producer runs ahead into the next tile while the
// consumers store the previous one.  Tiles are handed out round robin (persistent grid).
#pragma once
#include <cuda_fp16.h>
#include <string.h>
#include <type_traits>

#include "ptx.cuh"
#include "wgmma.cuh"

namespace b200 {

enum Layout { LAYOUT_K = 0, LAYOUT_MN = 1 };   // shared-memory layout of one operand (see above)

template <int KIND> struct KindTraits;
// B_LAYOUT: the layout of B for a row-major B, the default of the kernel's BL parameter (16-bit kinds: MN-major
// as stored; tf32 / int8: K-major, i.e. B^T).
template <> struct KindTraits<KIND_F16>  { static constexpr int ELEM = 2; static constexpr int B_LAYOUT = LAYOUT_MN; };
template <> struct KindTraits<KIND_FP16> { static constexpr int ELEM = 2; static constexpr int B_LAYOUT = LAYOUT_MN; };
template <> struct KindTraits<KIND_TF32> { static constexpr int ELEM = 4; static constexpr int B_LAYOUT = LAYOUT_K; };
template <> struct KindTraits<KIND_I8>   { static constexpr int ELEM = 1; static constexpr int B_LAYOUT = LAYOUT_K; };
template <> struct KindTraits<KIND_E4M3> { static constexpr int ELEM = 1; static constexpr int B_LAYOUT = LAYOUT_K; };
template <> struct KindTraits<KIND_E4M3E5M2> { static constexpr int ELEM = 1; static constexpr int B_LAYOUT = LAYOUT_K; };
template <> struct KindTraits<KIND_E5M2E4M3> { static constexpr int ELEM = 1; static constexpr int B_LAYOUT = LAYOUT_K; };

// Plane products issued per k-step.  Single: plain GEMM.  X3: a=a1+a2+a3, b likewise, all terms down
// to 2^-16 relative (a1b3, a3b1, a2b2, a1b2, a2b1, a1b1) — dropped terms are <= 2^-24.  X2: two planes,
// three terms, dropped a2b2 ~ 2^-16.
struct ProdSingle {
  static constexpr int N = 1, NPA = 1, NPB = 1;
  __host__ __device__ static constexpr int ia(int) { return 0; }
  __host__ __device__ static constexpr int ib(int) { return 0; }
};
struct ProdX3 {   // (ia,ib): (0,2) (2,0) (1,1) (0,1) (1,0) (0,0)
  static constexpr int N = 6, NPA = 3, NPB = 3;
  __host__ __device__ static constexpr int ia(int i) { return i == 1 ? 2 : (i == 2 || i == 4) ? 1 : 0; }
  __host__ __device__ static constexpr int ib(int i) { return i == 0 ? 2 : (i == 2 || i == 3) ? 1 : 0; }
};
struct ProdX2 {   // (0,1) (1,0) (0,0)
  static constexpr int N = 3, NPA = 2, NPB = 2;
  __host__ __device__ static constexpr int ia(int i) { return i == 1 ? 1 : 0; }
  __host__ __device__ static constexpr int ib(int i) { return i == 0 ? 1 : 0; }
};
// One plane, promoted: every chunk of TcParams::chunk_kb k-blocks starts a fresh wgmma accumulator that is added to the
// tile's fp32 running sum in registers (REGACC), as the split modes do.  The FP8 kernels use it with chunks of one k-block.
struct ProdPromoted : ProdSingle {};
template <class Prod> struct Promotes { static constexpr bool V = Prod::N > 1; };
template <> struct Promotes<ProdPromoted> { static constexpr bool V = true; };

struct TcParams {
  void* C;
  long long ldc;           // elements
  int M, N, K;
  int tiles_m, tiles_n;
  int group_m;             // rasterisation: tiles are walked m-fastest inside groups of group_m rows
  int vec_ok;              // C base and ldc allow 16-byte stores
  int a_plane_rows;        // row offset between stacked A planes (split modes), else 0
  int b_plane_rows;        // row offset between stacked B planes (split modes), else 0
  int chunk_kb;            // k-blocks per accumulation chunk (two-level accumulation), >= num_kb: off
  // Wave-quantisation tail: work items [0, full_tiles) are whole tiles; every later tile is cut
  // into `split` K-ranges processed by different CTAs in the last round and folded into C in
  // order (part p waits for flag == p on its 16-row strip, adds, then publishes p+1).
  int full_tiles, split;
  int* flags;              // [tail tile][consumer warp], zero between launches
  // Scaled split mode (B200_F32_F16X2): operands were multiplied by 2^-e(row) / 2^-e(col) before the
  // fp16 split; the epilogue multiplies back by 2^e(row) * 2^e(col), exact.  Null = no scaling.
  const float* row_max;    // [M] max |A(i,:)|
  union {
    const float* col_max;  // [N] max |B(:,j)|
    // EPI kernels (16-bit kinds, single plane, never scaled): the bias, n elements of the operand type (bf16 or fp16
    // bits), null = none.  It shares the slot so that TcParams, and with it every other kernel's code, is unchanged.
    const void* bias;
  };
  // General epilogue C = alpha * (A*B) + beta * C (cuBLAS semantics, cuda/MMult_cuBLAS_1.cpp:11-19); fp32, bf16 or
  // fp16 output (16-bit C is read exactly as fp32 and the result rounded once).  axpby == 0: alpha = 1 and
  // beta = accumulate (the two contracts the reference's harnesses use).
  float alpha, beta;
  int axpby;
  int accumulate;          // 1: C += A*B (every partial, including the first, is folded into C); fp32/int32 only
  int stream_c;            // 1: the split modes' single pass over C uses streaming (evict-first) stores
  int dbg_b_lbo, dbg_b_sbo;  // MN-major B descriptor strides, 0 = defaults (probe hook, see b200_gemm_debug_set_b_desc)
  int act;                 // EPI kernels: y = act(t + bias[col]) after the alpha / beta step; an EpiAct (ptx.cuh)
};

// Stacked kernels (gemm_tc_stacked_kernel) only: a second kernel argument, so that TcParams, and with it the code of
// every single-matrix kernel, is unchanged.  The operands are 3-D tensor maps (inner, rows, entry); a broadcast
// operand (stride 0) has one entry and is read at entry coordinate 0.  A grouped call is a stack whose A and C are
// broadcast: its groups are row ranges of both, and its entries are the B_g.  A K-grouped call is a stack whose A and B
// are broadcast: its groups are K ranges of both, and its entries are the C_g.
enum Stacking { STACK_NONE, STACK_BATCH, STACK_GROUP, STACK_KGROUP };
struct TcStack {
  int count;               // entries of a batch, or groups (1 .. kMaxGroups)
  int a_step, b_step;      // entry coordinate of A / B per entry: 1, or 0 for a broadcast operand
  long long stride_c;      // batch, K-grouped: elements between consecutive entries of C
  const int* offs;         // (K-)grouped: [count] cumulative ends of the groups, on the device (read after griddep_wait)
};

// REGACC (split-precision fp32 modes): the tensor core adds into its fp32 accumulator with truncation,
// so a long K chain drifts (error grows ~K).  K is cut into chunks of chunk_kb k-blocks; each chunk starts a
// fresh wgmma accumulator that is added, with a rounded fp32 add, to the tile's running sum in registers.
// AL / BL: layouts of A and B.  K-major A and MN-major B tiles are staged exactly as before this choice existed;
// an MN-major A tile is staged like an MN-major B tile (BM / 64 boxes of [BK rows x 128 B]) and a K-major B tile
// like a K-major A tile (BN rows of A_ROW_BYTES, SWIZZLE_128B or _64B), so byte counts are the same either way.
template <int KIND, int BN, int STAGES, class Prod, int A_ROW_BYTES, int AL = LAYOUT_K, int BL = KindTraits<KIND>::B_LAYOUT>
struct TcConfig {
  using T = KindTraits<KIND>;
  static constexpr bool A_MN = AL == LAYOUT_MN, B_MN = BL == LAYOUT_MN;
  static constexpr bool REGACC = Promotes<Prod>::V;       // Prod::N > 1, or ProdPromoted
  static constexpr int BM = 128;
  static constexpr int TILE_M = BM;                         // rows of C per work unit
  static constexpr int CONSUMERS = 2;                       // warpgroups, 64 rows each
  static constexpr int EPI_WARPS = 4 * CONSUMERS;           // warps that write C (16 rows each)
  static constexpr int BK = A_ROW_BYTES / T::ELEM;          // one swizzled row of K per stage
  static constexpr int A_PLANE = BM * A_ROW_BYTES;          // 16 KB (SW128) or 8 KB (SW64)
  static constexpr int A_SWZ = A_ROW_BYTES == 128 ? SWZ_128B : SWZ_64B;
  static constexpr int A_SBO = 8 * A_ROW_BYTES;             // K-major: 8-row core-matrix group stride
  static constexpr int MN_BOX_COLS = 128 / T::ELEM;         // MN-major: columns per 128-byte TMA box
  static constexpr int MN_BOX_BYTES = BK * 128;             // MN-major: one [BK rows x 128 B] box
  static constexpr int A_BOXES = A_MN ? BM / MN_BOX_COLS : 1;                // TMA boxes per A plane
  static constexpr int A_WG = A_MN ? MN_BOX_BYTES : 64 * A_ROW_BYTES;      // offset of the second consumer's rows
  static constexpr int B_BOX_COLS = B_MN ? MN_BOX_COLS : BN;               // B columns per TMA box
  static constexpr int B_BOX_ROWS = B_MN ? BK : BN;
  static constexpr int B_BOXES = BN / B_BOX_COLS;
  static constexpr int B_BOX_BYTES = B_MN ? MN_BOX_BYTES : BN * A_ROW_BYTES;
  static constexpr int B_PLANE = B_BOXES * B_BOX_BYTES;
  static constexpr int A_STAGE = Prod::NPA * A_PLANE;
  static constexpr int B_STAGE = Prod::NPB * B_PLANE;
  static constexpr int STAGE_BYTES = A_STAGE + B_STAGE;
  using MMA = Wgmma<KIND, BN, A_MN ? 1 : 0, B_MN ? 1 : 0>;
  static constexpr int MMA_K = MMA::K;
  static constexpr int MMAS_PER_STAGE = BK / MMA_K;
  // k advance per MMA: K-major: bytes inside the swizzled row; MN-major: k-rows of 128 B
  static constexpr int A_KADV = A_MN ? MMA_K * 128 : MMA_K * T::ELEM;
  static constexpr int B_KADV = B_MN ? MMA_K * 128 : MMA_K * T::ELEM;
  static constexpr int ACC = BN / 2;                        // accumulator registers per consumer thread
  static constexpr int SMEM_BYTES = 1024 /*align slack*/ + STAGES * STAGE_BYTES + 2 * STAGES * 8;
  static constexpr int THREADS = 128 * (1 + CONSUMERS);
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB dynamic shared memory of sm_90");
  static_assert(!REGACC || BN <= 128, "register accumulation keeps two 64 x BN fp32 tiles per consumer in registers");
  static_assert(T::ELEM == 2 || (!A_MN && !B_MN && Prod::NPA == 1 && Prod::NPB == 1 && A_ROW_BYTES == 128),
                "tf32 / int8: K-major A and B, single plane, 128-byte rows");
  static_assert(!B_MN || BN % MN_BOX_COLS == 0, "MN-major B is staged in 128-byte column blocks");
  static_assert(!A_MN || (A_BOXES == CONSUMERS && A_BOXES * MN_BOX_BYTES == A_PLANE),
                "MN-major A: one 64-column box per consumer warpgroup, the bytes of a K-major A plane");
  static_assert(B_PLANE == BN * A_ROW_BYTES, "a B plane holds BN x BK elements in either layout");
};

__device__ __forceinline__ void tile_coords(int t, int tiles_m, int tiles_n, int group_m, int& mb,
                                            int& nb) {
  const int per_group = group_m * tiles_n;
  const int g = t / per_group;
  const int first_m = g * group_m;
  const int rows = min(group_m, tiles_m - first_m);
  const int r = t - g * per_group;
  mb = first_m + r % rows;
  nb = r / rows;
}

// Scaled split mode (B200_F32_F16X2): exponent e with maxv * 2^-e in [0.5, 1) for every finite nonzero
// maxv (a subnormal maximum takes the exponent of its leading bit); 0 for zero, inf or NaN maxima.
// Range [-148, 128].
__host__ __device__ __forceinline__ int pow2_exp(float maxv) {
  uint32_t bits;
#ifdef __CUDA_ARCH__
  bits = __float_as_uint(maxv);
#else
  memcpy(&bits, &maxv, 4);
#endif
  const int ef = (int)((bits >> 23) & 0xFF);
  const uint32_t mant = bits & 0x7FFFFFu;          // a subnormal is mant * 2^-149
#ifdef __CUDA_ARCH__
  const int sub = (31 - __clz(mant | 1u)) - 148;
#else
  const int sub = (31 - __builtin_clz(mant | 1u)) - 148;
#endif
  return ef == 255 ? 0 : ef != 0 ? ef - 126 : mant != 0 ? sub : 0;
}
// 2^e as a float, e in [-126, 127]
__device__ __forceinline__ float exp2i(int e) { return __uint_as_float((uint32_t)(127 + e) << 23); }
// Pre-pass scaling x * 2^e, e in [-128, 148] (= -pow2_exp): two normal power-of-two factors.  Exact whenever
// the result is normal; a result below 2^-126 may be rounded twice, but every such value is below half the
// smallest fp16 subnormal and splits into zero planes either way.
__device__ __forceinline__ float scale_pow2(float x, int e) {
  const int h = e >> 1;
  return x * exp2i(h) * exp2i(e - h);
}
// F16X2 epilogue unscale: x * 2^e rounded once, for e in [-296, 256] (= e_row + e_col) and an accumulator x
// that is 0 or 2^-48 <= |x| < 2^32 (a sum of products of fp16 values below 1, each a multiple of 2^-48).
// x * 2^a with a = clamp(e, -78, 95) is exact and normal; the second factor 2^b, b = clamp(e - a, -126, 127),
// then rounds once.  b is clamped only where the result is below 2^-172 (rounds to 0 either way) or above
// 2^174 (overflows either way).  No factor is ever inf, so 0 stays 0.
__device__ __forceinline__ float mul_pow2(float x, int e) {
  const int a = max(min(e, 95), -78);
  const int b = max(min(e - a, 127), -126);
  return x * exp2i(a) * exp2i(b);
}

struct WorkItem { int tile, part, kb0, kb1; };
__device__ __forceinline__ WorkItem work_item(int w, const TcParams& p, int num_kb) {
  WorkItem it;
  if (w < p.full_tiles) { it.tile = w; it.part = 0; it.kb0 = 0; it.kb1 = num_kb; return it; }
  const int r = w - p.full_tiles;
  it.tile = p.full_tiles + r / p.split;
  it.part = r - (r / p.split) * p.split;
  it.kb0 = (int)((long long)num_kb * it.part / p.split);
  it.kb1 = (int)((long long)num_kb * (it.part + 1) / p.split);
  return it;
}

struct bf16_out {};   // tag: C stored as bf16 (RNE from the fp32 accumulator)
struct f16_out {};    // tag: C stored as fp16 (RNE from the fp32 accumulator; beyond 65504 rounds to +-inf)
struct s8_out {};     // tag: C stored as int8 through requant_s8 (TcParams::row_max = per-row scale,
                      // TcParams::col_max = per-row bias or null); int8 kernels only
struct e4m3_out {};   // tag: C stored as FP8 E4M3 bytes (FP8 kernels: cvt.rn.satfinite, see fp8_q8_tile)
struct e5m2_out {};   // tag: C stored as FP8 E5M2 bytes
template <typename OutT> struct OutBytes { static constexpr int V = 4; };
template <> struct OutBytes<bf16_out> { static constexpr int V = 2; };
template <> struct OutBytes<f16_out> { static constexpr int V = 2; };
template <> struct OutBytes<s8_out> { static constexpr int V = 1; };
template <> struct OutBytes<e4m3_out> { static constexpr int V = 1; };
template <> struct OutBytes<e5m2_out> { static constexpr int V = 1; };
template <typename OutT> struct Fp8Out { static constexpr bool V = false; };
template <> struct Fp8Out<e4m3_out> { static constexpr bool V = true; static constexpr float MAX = 448.f; };
template <> struct Fp8Out<e5m2_out> { static constexpr bool V = true; static constexpr float MAX = 57344.f; };

__device__ __forceinline__ uint32_t cvt_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ uint32_t cvt_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// One 16-bit C element (bf16 or fp16 bits) as fp32: exact.
template <typename OutT> __device__ __forceinline__ float c16_to_f32(uint32_t h) {
  if constexpr (std::is_same<OutT, f16_out>::value) return __half2float(__ushort_as_half((unsigned short)h));
  else return __uint_as_float(h << 16);
}

// One consumer thread's pair of adjacent columns (col, col + 1) of row `row` into C.
// ACT >= 0 (EPI kernels, fp32 / bf16 / fp16 C): after the alpha / beta step t = fma(beta, C, alpha * x), store
// act(t + b[e]); b = -0 when there is no bias (t + -0 is t for every t, the sign of zero included).
template <typename OutT, typename V, int ACT = -1>
__device__ __forceinline__ void store_pair(const TcParams& p, int row, int col, V v0, V v1, bool fold, bool l2_read,
                                           float al, float be, int re, const int (&ce)[2], float sc, float bi,
                                           float b0 = -0.f, float b1 = -0.f) {
  if (row >= p.M || col >= p.N) return;
  const bool both = col + 1 < p.N;
  if constexpr (std::is_same<OutT, float>::value) {
    float x[2] = {v0, v1};
    if (p.row_max != nullptr) { x[0] = mul_pow2(x[0], re + ce[0]); x[1] = mul_pow2(x[1], re + ce[1]); }
    if (p.axpby) { x[0] *= al; x[1] *= al; }
    float* dst = reinterpret_cast<float*>(p.C) + (long long)row * p.ldc + col;
    if (both && p.vec_ok) {
      if (fold) {
        // parts of a K-split tile were written by another SM in this launch: read them at L2, not through L1
        const float2 o = l2_read ? __ldcg(reinterpret_cast<const float2*>(dst)) : *reinterpret_cast<const float2*>(dst);
        if (p.axpby) { x[0] = fmaf(be, o.x, x[0]); x[1] = fmaf(be, o.y, x[1]); }
        else { x[0] += o.x; x[1] += o.y; }
      }
      if constexpr (ACT >= 0) { x[0] = epi_act<ACT>(__fadd_rn(x[0], b0)); x[1] = epi_act<ACT>(__fadd_rn(x[1], b1)); }
      if (p.stream_c) __stcs(reinterpret_cast<float2*>(dst), make_float2(x[0], x[1]));
      else *reinterpret_cast<float2*>(dst) = make_float2(x[0], x[1]);
    } else if constexpr (ACT >= 0) {
#pragma unroll
      for (int e = 0; e < 2; e++)
        if (e == 0 || both) {
          const float t = !fold ? x[e] : p.axpby ? fmaf(be, __ldcg(dst + e), x[e]) : x[e] + __ldcg(dst + e);
          dst[e] = epi_act<ACT>(__fadd_rn(t, e == 0 ? b0 : b1));
        }
    } else {
#pragma unroll
      for (int e = 0; e < 2; e++)
        if (e == 0 || both) dst[e] = !fold ? x[e] : p.axpby ? fmaf(be, __ldcg(dst + e), x[e]) : x[e] + __ldcg(dst + e);
    }
  } else if constexpr (std::is_same<OutT, int32_t>::value) {
    int32_t* dst = reinterpret_cast<int32_t*>(p.C) + (long long)row * p.ldc + col;
    int32_t x[2] = {v0, v1};
    if (both && p.vec_ok) {
      if (fold) { const int2 o = __ldcg(reinterpret_cast<const int2*>(dst)); x[0] += o.x; x[1] += o.y; }   // exact
      *reinterpret_cast<int2*>(dst) = make_int2(x[0], x[1]);
    } else {
#pragma unroll
      for (int e = 0; e < 2; e++)
        if (e == 0 || both) dst[e] = fold ? x[e] + __ldcg(dst + e) : x[e];
    }
  } else if constexpr (std::is_same<OutT, bf16_out>::value || std::is_same<OutT, f16_out>::value) {
    uint16_t* dst = reinterpret_cast<uint16_t*>(p.C) + (long long)row * p.ldc + col;
    float x[2] = {v0, v1};
    if (p.axpby) {            // general epilogue: round(fma(beta, float(C), alpha * AB)), C read only when beta != 0
      x[0] *= al; x[1] *= al;
      if (fold) {             // 16-bit C has no K-split tail: fold is beta != 0 here
        uint32_t o;
        if (both && p.vec_ok) o = *reinterpret_cast<const uint32_t*>(dst);
        else o = (uint32_t)dst[0] | (both ? (uint32_t)dst[1] << 16 : 0u);
        x[0] = fmaf(be, c16_to_f32<OutT>(o & 0xFFFFu), x[0]);
        x[1] = fmaf(be, c16_to_f32<OutT>(o >> 16), x[1]);
      }
    }
    if constexpr (ACT >= 0) { x[0] = epi_act<ACT>(__fadd_rn(x[0], b0)); x[1] = epi_act<ACT>(__fadd_rn(x[1], b1)); }
    const uint32_t w = std::is_same<OutT, f16_out>::value ? cvt_f16x2(x[0], x[1]) : cvt_bf16x2(x[0], x[1]);
    if (both && p.vec_ok) *reinterpret_cast<uint32_t*>(dst) = w;
    else {
      dst[0] = (uint16_t)w;
      if (both) dst[1] = (uint16_t)(w >> 16);
    }
  } else {
    uint8_t* dst = reinterpret_cast<uint8_t*>(p.C) + (long long)row * p.ldc + col;
    const uint32_t q0 = (uint32_t)requant_s8(v0, sc, bi, p.col_max != nullptr) & 0xFFu;
    const uint32_t q1 = (uint32_t)requant_s8(v1, sc, bi, p.col_max != nullptr) & 0xFFu;
    if (both && p.vec_ok) *reinterpret_cast<uint16_t*>(dst) = (uint16_t)(q0 | (q1 << 8));
    else {
      dst[0] = (uint8_t)q0;
      if (both) dst[1] = (uint8_t)q1;
    }
  }
}

// Bias + activation epilogue (EPI kernels) of one warp's 16 rows of a tile: the bias pair of each column pair is
// loaded once (one 4-byte load where the bias address allows) and shared by the thread's two rows.  ACT is the
// tile-uniform p.act, dispatched once per tile so that the unrolled store loop holds one activation only.
template <int KIND, typename OutT, int ACT, int BN>
__device__ __forceinline__ void epi_rows(const TcParams& p, const float (&acc)[BN / 2], int row0, int col0, bool fold,
                                         float al, float be) {
  using Bias16 = typename std::conditional<KIND == KIND_FP16, f16_out, bf16_out>::type;
  const uint16_t* bias = reinterpret_cast<const uint16_t*>(p.bias);
  const bool bias_vec = (reinterpret_cast<uintptr_t>(bias) & 3) == 0;
  const int ce[2] = {0, 0};
#pragma unroll
  for (int j = 0; j < BN / 8; j++) {
    const int col = col0 + 8 * j;
    float b[2] = {-0.f, -0.f};
    if (bias != nullptr && col < p.N) {
      uint32_t h;
      if (bias_vec && col + 1 < p.N) h = __ldg(reinterpret_cast<const unsigned int*>(bias + col));
      else h = (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(bias + col)) |
               (col + 1 < p.N ? (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(bias + col + 1)) << 16 : 0u);
      b[0] = c16_to_f32<Bias16>(h & 0xFFFFu);
      b[1] = c16_to_f32<Bias16>(h >> 16);
    }
#pragma unroll
    for (int h = 0; h < 2; h++)
      store_pair<OutT, float, ACT>(p, row0 + 8 * h, col, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], fold, false, al, be,
                                   0, ce, 0.f, 0.f, b[0], b[1]);
  }
}

// EPI: the bias / activation epilogue (16-bit kinds, single plane, float / bf16_out / f16_out C).  Its kernels never
// take the K-split tail (launch_tc sets split = 1): the activation must see the complete sum.
template <int KIND, int BN, int STAGES, typename OutT, class Prod, int A_ROW_BYTES, int AL = LAYOUT_K,
          int BL = KindTraits<KIND>::B_LAYOUT, bool EPI = false>
__global__ void __launch_bounds__((TcConfig<KIND, BN, STAGES, Prod, A_ROW_BYTES, AL, BL>::THREADS), 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const TcParams p) {
  using Cfg = TcConfig<KIND, BN, STAGES, Prod, A_ROW_BYTES, AL, BL>;
  using MMA = typename Cfg::MMA;
  using Acc = typename MMA::Acc;
  static_assert(!EPI || (KindTraits<KIND>::ELEM == 2 && !Cfg::REGACC &&
                         (std::is_same<OutT, float>::value || OutBytes<OutT>::V == 2)),
                "bias / activation epilogue: 16-bit single-plane kinds with fp32 or 16-bit C");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // swizzle atoms need 1 KB
  const uint32_t sA = smem_base;
  const uint32_t sB = sA + STAGES * Cfg::A_STAGE;
  const uint32_t bar_full = sB + STAGES * Cfg::B_STAGE;
  const uint32_t bar_empty = bar_full + 8 * STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; i++) {
      mbar_init(bar_full + 8 * i, 1);
      mbar_init(bar_empty + 8 * i, Cfg::CONSUMERS);          // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  // PDL: everything above may overlap the tail of the previous kernel in the stream; nothing below
  // (operand loads, C stores) may.
  griddep_launch();
  griddep_wait();

  const int num_tiles = p.tiles_m * p.tiles_n;
  const int num_items = p.full_tiles + (num_tiles - p.full_tiles) * p.split;
  const int num_kb = (p.K + Cfg::BK - 1) / Cfg::BK;

  if (warp < 4) {
    // ===================== TMA producer (warpgroup 0) =====================
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int w = blockIdx.x; w < num_items; w += gridDim.x) {
        const WorkItem it = work_item(w, p, num_kb);
        int mb, nb;
        tile_coords(it.tile, p.tiles_m, p.tiles_n, p.group_m, mb, nb);
        const int m0 = mb * Cfg::BM, n0 = nb * BN;
        for (int kb = it.kb0; kb < it.kb1; kb++) {
          mbar_wait(bar_empty + 8 * s, ph ^ 1);
          const uint32_t full = bar_full + 8 * s;
          mbar_arrive_expect_tx(full, Cfg::STAGE_BYTES);
          if constexpr (Cfg::A_MN) {                  // A^T (k x m): one 64-column box per consumer
#pragma unroll
            for (int pa = 0; pa < Prod::NPA; pa++)
#pragma unroll
              for (int j = 0; j < Cfg::A_BOXES; j++)
                tma_load_2d(sA + s * Cfg::A_STAGE + pa * Cfg::A_PLANE + j * Cfg::MN_BOX_BYTES, &tmA, full,
                            m0 + j * Cfg::MN_BOX_COLS, pa * p.a_plane_rows + kb * Cfg::BK);
          } else {
#pragma unroll
            for (int pa = 0; pa < Prod::NPA; pa++)
              tma_load_2d(sA + s * Cfg::A_STAGE + pa * Cfg::A_PLANE, &tmA, full, kb * Cfg::BK, pa * p.a_plane_rows + m0);
          }
          if constexpr (!Cfg::B_MN) {                 // B^T (n x k): one box of BN rows per plane
            if constexpr (Prod::NPB == 1) {
              tma_load_2d(sB + s * Cfg::B_STAGE, &tmB, full, kb * Cfg::BK, n0);
            } else {
#pragma unroll
              for (int pb = 0; pb < Prod::NPB; pb++)
                tma_load_2d(sB + s * Cfg::B_STAGE + pb * Cfg::B_PLANE, &tmB, full, kb * Cfg::BK, pb * p.b_plane_rows + n0);
            }
          } else {
#pragma unroll
            for (int pb = 0; pb < Prod::NPB; pb++)
#pragma unroll
              for (int j = 0; j < Cfg::B_BOXES; j++)
                tma_load_2d(sB + s * Cfg::B_STAGE + pb * Cfg::B_PLANE + j * Cfg::B_BOX_BYTES, &tmB, full,
                            n0 + j * Cfg::B_BOX_COLS, pb * p.b_plane_rows + kb * Cfg::BK);
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers (warpgroups 1 and 2): MMA chain + epilogue =====================
    setmaxnreg_inc<232>();
    const int cw = warp / 4 - 1;                    // consumer warpgroup: rows [64 cw, 64 cw + 64) of the tile
    const int ew = warp - 4;                        // consumer warp 0..7: 16 rows each
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const uint32_t b_lbo = p.dbg_b_lbo ? (uint32_t)p.dbg_b_lbo : (uint32_t)Cfg::B_BOX_BYTES;
    const uint32_t b_sbo = p.dbg_b_sbo ? (uint32_t)p.dbg_b_sbo : 1024u;
    int s = 0;
    uint32_t ph = 0;
    Acc acc[Cfg::ACC];
    float sum[Cfg::REGACC ? Cfg::ACC : 1];
    for (int w = blockIdx.x; w < num_items; w += gridDim.x) {
      const WorkItem it = work_item(w, p, num_kb);
      int mb, nb;
      tile_coords(it.tile, p.tiles_m, p.tiles_n, p.group_m, mb, nb);
      const int m0 = mb * Cfg::BM, n0 = nb * BN;
      const int chunk = Cfg::REGACC ? p.chunk_kb : it.kb1 - it.kb0;
      for (int c0 = it.kb0; c0 < it.kb1; c0 += chunk) {
        const int c1 = min(c0 + chunk, it.kb1);
        int prev = -1;
        for (int kb = c0; kb < c1; kb++) {
          mbar_wait(bar_full + 8 * s, ph);
          const uint32_t a0 = sA + s * Cfg::A_STAGE + cw * Cfg::A_WG;
          const uint32_t b0 = sB + s * Cfg::B_STAGE;
          wgmma_fence();
#pragma unroll
          for (int pr = 0; pr < Prod::N; pr++) {
#pragma unroll
            for (int k = 0; k < Cfg::MMAS_PER_STAGE; k++) {
              // K-major: SBO = 8-row group stride, LBO unused; MN-major: LBO = column-block stride, SBO = 8 k-rows
              uint64_t ad, bd;
              if constexpr (Cfg::A_MN)
                ad = make_sdesc(a0 + Prod::ia(pr) * Cfg::A_PLANE + k * Cfg::A_KADV, Cfg::MN_BOX_BYTES, 1024, SWZ_128B);
              else
                ad = make_sdesc(a0 + Prod::ia(pr) * Cfg::A_PLANE + k * Cfg::A_KADV, 16, Cfg::A_SBO, Cfg::A_SWZ);
              if constexpr (Cfg::B_MN)
                bd = make_sdesc(b0 + Prod::ib(pr) * Cfg::B_PLANE + k * Cfg::B_KADV, b_lbo, b_sbo, SWZ_128B);
              else if constexpr (Prod::NPB == 1)
                bd = make_sdesc(b0 + k * Cfg::B_KADV, 16, Cfg::A_SBO, Cfg::A_SWZ);
              else
                bd = make_sdesc(b0 + Prod::ib(pr) * Cfg::B_PLANE + k * Cfg::B_KADV, 16, Cfg::A_SBO, Cfg::A_SWZ);
              MMA::mma(acc, ad, bd, ((kb - c0) | k | pr) != 0 ? 1u : 0u);
            }
          }
          wgmma_commit();
          wgmma_wait<1>();                            // the previous k-block's products retired: its stage is free
          if (prev >= 0 && wg_leader) mbar_arrive(bar_empty + 8 * prev);
          prev = s;
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (prev >= 0 && wg_leader) mbar_arrive(bar_empty + 8 * prev);
        if constexpr (Cfg::REGACC) {
#pragma unroll
          for (int i = 0; i < Cfg::ACC; i++) sum[i] = c0 == it.kb0 ? acc[i] : __fadd_rn(sum[i], acc[i]);
        }
      }

      // ---- this warp's 16 rows of the tile into C ----
      int* flag = p.flags + (it.tile - p.full_tiles) * Cfg::EPI_WARPS + ew;
      if (it.part > 0) {                               // K-split tail: wait until parts < it.part are in C
        if (lane == 0) {
          const long long t0 = clock64();
          while (true) {
            int v;
            asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
            if (v == it.part) break;
            if (clock64() - t0 > 4000000000LL) { asm volatile("trap;"); }
          }
        }
        __syncwarp();
      }
      // beta * C is read by part 0 only; later K parts add alpha * partial to what is already there
      const bool fold = p.accumulate != 0 || it.part > 0 || (p.axpby && p.beta != 0.f);
      const float al = p.axpby ? p.alpha : 1.f;
      const float be = (p.axpby && it.part == 0) ? p.beta : 1.f;
      const int row0 = m0 + ew * 16 + (lane >> 2);
      const int col0 = n0 + 2 * (lane & 3);
      int re[2] = {0, 0};
      float sc[2] = {0.f, 0.f}, bi[2] = {0.f, 0.f};
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int row = row0 + 8 * h;
        if (row < p.M) {
          if constexpr (std::is_same<OutT, s8_out>::value) {
            sc[h] = __ldg(p.row_max + row);
            if (p.col_max != nullptr) bi[h] = __ldg(p.col_max + row);
          } else if (p.row_max != nullptr) {
            re[h] = pow2_exp(__ldg(p.row_max + row));
          }
        }
      }
      if constexpr (EPI) {
        switch (p.act) {
          case ACT_RELU: epi_rows<KIND, OutT, ACT_RELU, BN>(p, acc, row0, col0, fold, al, be); break;
          case ACT_GELU: epi_rows<KIND, OutT, ACT_GELU, BN>(p, acc, row0, col0, fold, al, be); break;
          case ACT_GELU_TANH: epi_rows<KIND, OutT, ACT_GELU_TANH, BN>(p, acc, row0, col0, fold, al, be); break;
          default: epi_rows<KIND, OutT, ACT_NONE, BN>(p, acc, row0, col0, fold, al, be); break;
        }
      } else {
#pragma unroll
        for (int j = 0; j < BN / 8; j++) {
          const int col = col0 + 8 * j;
          int ce[2] = {0, 0};
          if (!std::is_same<OutT, s8_out>::value && p.col_max != nullptr) {
#pragma unroll
            for (int e = 0; e < 2; e++)
              if (col + e < p.N) ce[e] = pow2_exp(__ldg(p.col_max + col + e));
          }
#pragma unroll
          for (int h = 0; h < 2; h++) {
            if constexpr (Cfg::REGACC)
              store_pair<OutT>(p, row0 + 8 * h, col, sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1], fold, it.part > 0, al, be,
                               re[h], ce, sc[h], bi[h]);
            else
              store_pair<OutT>(p, row0 + 8 * h, col, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], fold, it.part > 0, al,
                               be, re[h], ce, sc[h], bi[h]);
          }
        }
      }
      if (w >= p.full_tiles && p.split > 1) {          // publish this part (the last one re-arms the flag)
        __threadfence();
        __syncwarp();
        if (lane == 0) {
          const int nv = it.part + 1 == p.split ? 0 : it.part + 1;
          asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(flag), "r"(nv) : "memory");
        }
      }
    }
  }
}

// ---- split-precision fp32 GEMM with the epilogue behind the next tile's MMAs (gemm_tc_split_kernel) -------------------
// k-blocks of the next work item issued before a tile's store, which is cut into as many slices (2 .. 4, < STAGES)
constexpr int kSplitEpiOverlap = 3;

// wgmma.wait_group with an argument that is a constant after unrolling (0 .. 3)
__device__ __forceinline__ void wgmma_wait_upto(int n) {
  switch (n) {
    case 0: wgmma_wait<0>(); break;
    case 1: wgmma_wait<1>(); break;
    case 2: wgmma_wait<2>(); break;
    default: wgmma_wait<3>(); break;
  }
}

// One k-block's plane products into acc (gemm_tc_kernel's chain): wait for stage s, issue, commit.  `first`: the first
// k-block of a chunk, whose first product starts the accumulator from zero.
template <class Cfg, class Prod>
__device__ __forceinline__ void split_issue_kblock(float (&acc)[Cfg::ACC], uint32_t sA, uint32_t sB, uint32_t bar_full,
                                                   int s, uint32_t ph, int cw, uint32_t b_lbo, uint32_t b_sbo,
                                                   bool first) {
  using MMA = typename Cfg::MMA;
  mbar_wait(bar_full + 8 * s, ph);
  const uint32_t a0 = sA + s * Cfg::A_STAGE + cw * Cfg::A_WG;
  const uint32_t b0 = sB + s * Cfg::B_STAGE;
  wgmma_fence();
#pragma unroll
  for (int pr = 0; pr < Prod::N; pr++) {
#pragma unroll
    for (int k = 0; k < Cfg::MMAS_PER_STAGE; k++) {
      uint64_t ad, bd;
      if constexpr (Cfg::A_MN)
        ad = make_sdesc(a0 + Prod::ia(pr) * Cfg::A_PLANE + k * Cfg::A_KADV, Cfg::MN_BOX_BYTES, 1024, SWZ_128B);
      else
        ad = make_sdesc(a0 + Prod::ia(pr) * Cfg::A_PLANE + k * Cfg::A_KADV, 16, Cfg::A_SBO, Cfg::A_SWZ);
      if constexpr (Cfg::B_MN)
        bd = make_sdesc(b0 + Prod::ib(pr) * Cfg::B_PLANE + k * Cfg::B_KADV, b_lbo, b_sbo, SWZ_128B);
      else
        bd = make_sdesc(b0 + Prod::ib(pr) * Cfg::B_PLANE + k * Cfg::B_KADV, 16, Cfg::A_SBO, Cfg::A_SWZ);
      MMA::mma(acc, ad, bd, ((first ? 0 : 1) | k | pr) != 0 ? 1u : 0u);
    }
  }
  wgmma_commit();
}

// Whether work item w's tile is stored by split_store_plain: a whole tile (no K split) inside M x N whose C takes plain
// 8-byte stores of the unscaled sum (no fold, alpha / beta or streaming).
template <class Cfg>
__device__ __forceinline__ bool split_tile_plain(const TcParams& p, int w, int num_kb) {
  const WorkItem it = work_item(w, p, num_kb);
  int mb, nb;
  tile_coords(it.tile, p.tiles_m, p.tiles_n, p.group_m, mb, nb);
  return w < p.full_tiles && (mb + 1) * Cfg::BM <= p.M && (nb + 1) * 128 <= p.N && p.vec_ok && !p.accumulate &&
         !p.axpby && !p.stream_c && p.row_max != nullptr;
}

// One consumer warp's 16 rows of a split_tile_plain work item (its fp32 running sum `sum`) into C: per column pair
// the two exponents, then the pair of both rows unscaled by mul_pow2 as store_pair does it and stored, with no per-pair
// branch.  The 16 column groups go in kSplitEpiOverlap slices.  OVERLAP: the next item's first kSplitEpiOverlap
// k-blocks are in flight from stage st0 on; after slice i the first i + 1 of them are retired and their stages
// released, so a k-block stays queued on the tensor pipe while each slice is stored, and none is left after the last.
template <class Cfg, int STAGES, bool OVERLAP>
__device__ __forceinline__ void split_store_plain(const TcParams& p, const float (&sum)[Cfg::ACC], int w, int num_kb,
                                                  int ew, int lane, int st0, uint32_t bar_empty, bool wg_leader) {
  constexpr int J = 128 / 8, D = kSplitEpiOverlap;
  const WorkItem it = work_item(w, p, num_kb);
  int mb, nb;
  tile_coords(it.tile, p.tiles_m, p.tiles_n, p.group_m, mb, nb);
  const int row0 = mb * Cfg::BM + ew * 16 + (lane >> 2);
  const int col0 = nb * 128 + 2 * (lane & 3);
  const int re[2] = {pow2_exp(__ldg(p.row_max + row0)), pow2_exp(__ldg(p.row_max + row0 + 8))};
  const float* const cmax = p.col_max + col0;
  float* const c_row = reinterpret_cast<float*>(p.C) + (long long)row0 * p.ldc + col0;
#pragma unroll
  for (int i = 0; i < D; i++) {
#pragma unroll
    for (int j = J * i / D; j < J * (i + 1) / D; j++) {
      const int ce0 = cmax != nullptr ? pow2_exp(__ldg(cmax + 8 * j)) : 0;
      const int ce1 = cmax != nullptr ? pow2_exp(__ldg(cmax + 8 * j + 1)) : 0;
#pragma unroll
      for (int h = 0; h < 2; h++)
        *reinterpret_cast<float2*>(c_row + 8 * h * p.ldc + 8 * j) =
            make_float2(mul_pow2(sum[4 * j + 2 * h], re[h] + ce0), mul_pow2(sum[4 * j + 2 * h + 1], re[h] + ce1));
    }
    if constexpr (OVERLAP) {
      wgmma_wait_upto(D - 1 - i);
      if (wg_leader) mbar_arrive(bar_empty + 8 * ((st0 + i) % STAGES));
    }
  }
}

// Every other work item: gemm_tc_kernel's epilogue (K-split wait and publish, store_pair per column pair).
template <class Cfg>
__device__ __forceinline__ void split_store_general(const TcParams& p, const float (&sum)[Cfg::ACC], int w, int num_kb,
                                                    int ew, int lane) {
  const WorkItem it = work_item(w, p, num_kb);
  int mb, nb;
  tile_coords(it.tile, p.tiles_m, p.tiles_n, p.group_m, mb, nb);
  int* flag = p.flags + (it.tile - p.full_tiles) * Cfg::EPI_WARPS + ew;
  if (it.part > 0) {                               // K-split tail: wait until parts < it.part are in C
    if (lane == 0) {
      const long long t0 = clock64();
      while (true) {
        int v;
        asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
        if (v == it.part) break;
        if (clock64() - t0 > 4000000000LL) { asm volatile("trap;"); }
      }
    }
    __syncwarp();
  }
  // beta * C is read by part 0 only; later K parts add alpha * partial to what is already there
  const bool fold = p.accumulate != 0 || it.part > 0 || (p.axpby && p.beta != 0.f);
  const float al = p.axpby ? p.alpha : 1.f;
  const float be = (p.axpby && it.part == 0) ? p.beta : 1.f;
  const int row0 = mb * Cfg::BM + ew * 16 + (lane >> 2);
  const int col0 = nb * 128 + 2 * (lane & 3);
  int re[2] = {0, 0};
#pragma unroll
  for (int h = 0; h < 2; h++)
    if (row0 + 8 * h < p.M && p.row_max != nullptr) re[h] = pow2_exp(__ldg(p.row_max + row0 + 8 * h));
#pragma unroll
  for (int j = 0; j < 128 / 8; j++) {
    const int col = col0 + 8 * j;
    int ce[2] = {0, 0};
    if (p.col_max != nullptr) {
#pragma unroll
      for (int e = 0; e < 2; e++)
        if (col + e < p.N) ce[e] = pow2_exp(__ldg(p.col_max + col + e));
    }
#pragma unroll
    for (int h = 0; h < 2; h++)
      store_pair<float>(p, row0 + 8 * h, col, sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1], fold, it.part > 0, al, be,
                        re[h], ce, 0.f, 0.f);
  }
  if (w >= p.full_tiles && p.split > 1) {          // publish this part (the last one re-arms the flag)
    __threadfence();
    __syncwarp();
    if (lane == 0) {
      const int nv = it.part + 1 == p.split ? 0 : it.part + 1;
      asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(flag), "r"(nv) : "memory");
    }
  }
}

// The split-precision fp32 kernel (F16X2): gemm_tc_kernel's producer, stage ring, descriptors, MMA chain, chunked fold
// into the register running sum and K-split tail, for fp32 C in 128 x 128 tiles, with each work item's epilogue
// run behind the next item's first k-blocks.  When item w's last chunk is folded into `sum`, the consumers issue the
// CTA's next item's first kSplitEpiOverlap k-blocks into `acc` (its first chunk starts from zero, so acc holds nothing
// of w) and store w from `sum` while the tensor cores run them.  The CTA's last item, and a tile that needs
// store_pair's general store (edge tiles, fold, alpha / beta, streaming stores, K parts), are stored before any further
// issue, as gemm_tc_kernel does.  Every product, fold and unscaling is gemm_tc_kernel's, so C is the same bit for bit.
// A kernel of its own so that gemm_tc_kernel keeps its code (DESIGN.md §4.1, "Why a kernel of its own").
template <int KIND, int BN, int STAGES, class Prod, int A_ROW_BYTES, int AL, int BL>
__global__ void __launch_bounds__((TcConfig<KIND, BN, STAGES, Prod, A_ROW_BYTES, AL, BL>::THREADS), 1)
gemm_tc_split_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const TcParams p) {
  using Cfg = TcConfig<KIND, BN, STAGES, Prod, A_ROW_BYTES, AL, BL>;
  constexpr int D = kSplitEpiOverlap;
  static_assert(Cfg::REGACC && Prod::N > 1 && BN == 128, "split-precision modes: register running sum, 128-wide tiles");
  static_assert(D >= 2 && D <= 4 && D < STAGES, "the deferred epilogue holds D stages while the producer refills the rest");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // swizzle atoms need 1 KB
  const uint32_t sA = smem_base;
  const uint32_t sB = sA + STAGES * Cfg::A_STAGE;
  const uint32_t bar_full = sB + STAGES * Cfg::B_STAGE;
  const uint32_t bar_empty = bar_full + 8 * STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; i++) {
      mbar_init(bar_full + 8 * i, 1);
      mbar_init(bar_empty + 8 * i, Cfg::CONSUMERS);          // one arrive per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  // PDL: everything above may overlap the tail of the previous kernel in the stream; nothing below may.
  griddep_launch();
  griddep_wait();

  const int num_tiles = p.tiles_m * p.tiles_n;
  const int num_items = p.full_tiles + (num_tiles - p.full_tiles) * p.split;
  const int num_kb = (p.K + Cfg::BK - 1) / Cfg::BK;

  if (warp < 4) {
    // ===================== TMA producer (warpgroup 0), as in gemm_tc_kernel =====================
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int w = blockIdx.x; w < num_items; w += gridDim.x) {
        const WorkItem it = work_item(w, p, num_kb);
        int mb, nb;
        tile_coords(it.tile, p.tiles_m, p.tiles_n, p.group_m, mb, nb);
        const int m0 = mb * Cfg::BM, n0 = nb * BN;
        for (int kb = it.kb0; kb < it.kb1; kb++) {
          mbar_wait(bar_empty + 8 * s, ph ^ 1);
          const uint32_t full = bar_full + 8 * s;
          mbar_arrive_expect_tx(full, Cfg::STAGE_BYTES);
          if constexpr (Cfg::A_MN) {
#pragma unroll
            for (int pa = 0; pa < Prod::NPA; pa++)
#pragma unroll
              for (int j = 0; j < Cfg::A_BOXES; j++)
                tma_load_2d(sA + s * Cfg::A_STAGE + pa * Cfg::A_PLANE + j * Cfg::MN_BOX_BYTES, &tmA, full,
                            m0 + j * Cfg::MN_BOX_COLS, pa * p.a_plane_rows + kb * Cfg::BK);
          } else {
#pragma unroll
            for (int pa = 0; pa < Prod::NPA; pa++)
              tma_load_2d(sA + s * Cfg::A_STAGE + pa * Cfg::A_PLANE, &tmA, full, kb * Cfg::BK, pa * p.a_plane_rows + m0);
          }
          if constexpr (!Cfg::B_MN) {
#pragma unroll
            for (int pb = 0; pb < Prod::NPB; pb++)
              tma_load_2d(sB + s * Cfg::B_STAGE + pb * Cfg::B_PLANE, &tmB, full, kb * Cfg::BK, pb * p.b_plane_rows + n0);
          } else {
#pragma unroll
            for (int pb = 0; pb < Prod::NPB; pb++)
#pragma unroll
              for (int j = 0; j < Cfg::B_BOXES; j++)
                tma_load_2d(sB + s * Cfg::B_STAGE + pb * Cfg::B_PLANE + j * Cfg::B_BOX_BYTES, &tmB, full,
                            n0 + j * Cfg::B_BOX_COLS, pb * p.b_plane_rows + kb * Cfg::BK);
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers (warpgroups 1 and 2): MMA chain + deferred epilogue =====================
    setmaxnreg_inc<232>();
    const int cw = warp / 4 - 1;                    // consumer warpgroup: rows [64 cw, 64 cw + 64) of the tile
    const int ew = warp - 4;                        // consumer warp 0..7: 16 rows each
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const uint32_t b_lbo = p.dbg_b_lbo ? (uint32_t)p.dbg_b_lbo : (uint32_t)Cfg::B_BOX_BYTES;
    const uint32_t b_sbo = p.dbg_b_sbo ? (uint32_t)p.dbg_b_sbo : 1024u;
    int s = 0;
    uint32_t ph = 0;
    float acc[Cfg::ACC];
    float sum[Cfg::ACC];
    // Every work item's first chunk is at least min(chunk_kb, num_kb / split) k-blocks long (a K part has at least
    // num_kb / split), so this says whether each one has the D k-blocks a deferred store runs behind.
    const bool hide = min(p.chunk_kb, num_kb / p.split) >= D;
    int skip = 0;                                   // k-blocks of this item issued behind the previous item's store
    for (int w = blockIdx.x; w < num_items; w += gridDim.x) {
      const WorkItem it = work_item(w, p, num_kb);
      for (int c0 = it.kb0; c0 < it.kb1; c0 += p.chunk_kb) {
        const int c1 = min(c0 + p.chunk_kb, it.kb1);
        int prev = -1;
        for (int kb = c0 + skip; kb < c1; kb++) {
          split_issue_kblock<Cfg, Prod>(acc, sA, sB, bar_full, s, ph, cw, b_lbo, b_sbo, kb == c0);
          wgmma_wait<1>();                            // the previous k-block's products retired: its stage is free
          if (prev >= 0 && wg_leader) mbar_arrive(bar_empty + 8 * prev);
          prev = s;
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
        skip = 0;
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (prev >= 0 && wg_leader) mbar_arrive(bar_empty + 8 * prev);
#pragma unroll
        for (int i = 0; i < Cfg::ACC; i++) sum[i] = c0 == it.kb0 ? acc[i] : __fadd_rn(sum[i], acc[i]);
      }
      // ---- this warp's 16 rows of the tile into C: behind the next item's first D k-blocks where possible ----
      if (split_tile_plain<Cfg>(p, w, num_kb)) {
        if (hide && w + (int)gridDim.x < num_items) {
          const int st0 = s;
#pragma unroll
          for (int i = 0; i < D; i++) {
            split_issue_kblock<Cfg, Prod>(acc, sA, sB, bar_full, s, ph, cw, b_lbo, b_sbo, i == 0);
            if (++s == STAGES) { s = 0; ph ^= 1; }
          }
          split_store_plain<Cfg, STAGES, true>(p, sum, w, num_kb, ew, lane, st0, bar_empty, wg_leader);
          skip = D;
        } else {
          split_store_plain<Cfg, STAGES, false>(p, sum, w, num_kb, ew, lane, 0, bar_empty, wg_leader);
        }
      } else {
        split_store_general<Cfg>(p, sum, w, num_kb, ew, lane);
      }
    }
  }
}

// ---- the entry of a work tile of the stacked kernels (gemm_tc_stacked_kernel, gemm_tc_fp8_kernel with STACK) -----------
struct StackEntry {
  int tile0, tiles_m;      // the entry's first work tile and its tile rows (tile_coords)
  int a_row, a_entry;      // A: row of the entry's first row, entry coordinate
  int b_entry;             // B: entry coordinate
  int M;                   // rows of the entry's C
  long long c_off;         // elements from C to the entry's first row
  int k0, k_len;           // KGROUP: the group's first K row and its k_g
  int entry;               // the entry's index (batch entry or group), whatever its operands' entry coordinates
};
// The entry of work tile `tile`.  grp_end / grp_tile: the GROUP kernels' tables (group_table), grp_end the KGROUP
// kernels' K ends, else unused.
template <int STACK>
__device__ __forceinline__ StackEntry stack_entry(int tile, const TcParams& p, const TcStack& st, const int* grp_end,
                                                  const int* grp_tile) {
  StackEntry se;
  int e;
  if constexpr (STACK == STACK_GROUP) {
    e = group_of(grp_tile, st.count, tile / p.tiles_n);
    se.tile0 = grp_tile[e] * p.tiles_n;
    se.tiles_m = grp_tile[e + 1] - grp_tile[e];
    se.a_row = grp_end[e];
    se.M = grp_end[e + 1] - grp_end[e];
    se.c_off = (long long)grp_end[e] * p.ldc;
  } else {
    const int per_entry = p.tiles_m * p.tiles_n;
    e = tile / per_entry;
    se.tile0 = e * per_entry;
    se.tiles_m = p.tiles_m;
    se.a_row = 0;
    se.M = p.M;
    se.c_off = (long long)e * st.stride_c;
  }
  if constexpr (STACK == STACK_KGROUP) {
    se.k0 = grp_end[e];
    se.k_len = grp_end[e + 1] - grp_end[e];
  } else {
    se.k0 = 0;
    se.k_len = p.K;
  }
  se.a_entry = e * st.a_step;
  se.b_entry = e * st.b_step;
  se.entry = e;
  return se;
}

// ---- FP8 GEMM (torch._scaled_mm) ---------------------------------------------------------------------------------------
// C = round_out((acc * sa_i) * sb_j + bias_j), each step one fp32 round-to-nearest operation (explicit intrinsics: no
// FMA contraction).  acc is op(A) op(B) of the FP8 operands: with ProdSingle one wgmma accumulator over all of K
// (fast accumulation); with ProdPromoted every chunk of p.chunk_kb k-blocks (the host passes one k-block, 128 elements)
// starts a fresh accumulator that is added, rounded, to the tile's fp32 running sum in registers.  The scales are fp32
// on the device, read here and never by the host: row i of A takes a[i * a_step] and column j of B b[j * b_step], a step
// of 0 for one tensorwise scale and 1 for a vector.  It is a kernel of its own (a second argument, no K split, no
// alpha / beta) so that gemm_tc_kernel and TcParams keep their code; its producer and MMA chain are gemm_tc_kernel's for
// K-major A and B, and its store is store_pair's bias path.
struct TcScale {
  const float* a;          // [m] or [1]
  const float* b;          // [n] or [1]
  int a_step, b_step;      // 0 = tensorwise, 1 = one scale per row of A / column of B
  const void* bias;        // [n] of C's type (bf16 / fp16 bits, or fp32; bf16 for an FP8 C), null = none
};

// Blockwise scales (BLOCKWISE kernels, torch._scaled_mm's 1 x 128 / 128 x 128 recipes): k-block kb (K elements
// [128 kb, 128 kb + 128)) of row i takes sa = a[ia * a_row + kb * a_kb] and of column j sb = b[kb * b_kb + jb * b_col],
// ia = i for a_blk = 1 and i / 128 for 128, jb likewise; strides in elements, any non-negative value (0 broadcasts).
// The promotion of that k-block is sum = fma(acc_kb, rn(sa * sb), sum) from sum = +0, and the store is store_pair's
// bias path with no further scaling.  Its own argument type, so that TcScale, and the existing FP8 kernels, keep
// their layout and code.
struct TcBlockScale {
  const float* a;
  const float* b;
  long long a_row, a_kb;   // scale_a strides: per row (a_blk = 1) or 128-row block (128), per k-block
  long long b_kb, b_col;   // scale_b strides: per k-block, per column (b_blk = 1) or 128-column block (128)
  int a_blk, b_blk;        // 1 or 128, never both 128
  const void* bias;        // as TcScale::bias
};
// Stacked FP8 kernels (STACK_GROUP / STACK_BATCH, torch._scaled_grouped_mm): rowwise scales only (a_step = b_step = 1,
// no bias), the stack, and the scales' element strides between entries.  Entry e's row i takes a[i_global] (grouped:
// the row of the stacked A) or a[e * a_entry_stride + i] (batch), and its column j b[e * b_entry_stride + j]: scales
// follow the entry index, so a broadcast operand (entry coordinate 0) still gets each entry's own scales.
struct TcStackScale : TcScale {
  TcStack st;
  long long a_entry_stride, b_entry_stride;
};
// Stacked blockwise FP8 kernels (BLOCKWISE with STACK_GROUP / STACK_BATCH): TcBlockScale's indexing inside each entry,
// no bias, plus the stack and the scales' element strides between entries.  Entry e's k-block kb takes, for row i,
// a[(end_{e-1} + i) * a_row + kb * a_kb] (grouped: the row of the stacked A, a_blk = 1 only) or
// a[e * a_entry_stride + ia * a_row + kb * a_kb] (batch), and for column j b[e * b_entry_stride + kb * b_kb + jb * b_col].
struct TcStackBlockScale : TcBlockScale {
  TcStack st;
  long long a_entry_stride, b_entry_stride;
};
// FP8 output (OutT e4m3_out / e5m2_out, single-matrix kernels): each element's fp32 value v is the existing kernels'
// value before round_out (tensorwise / rowwise: act(rn(rn(rn(acc * sa_i) * sb_j) + bias_j)); blockwise:
// act(rn(sum + bias_j))), with a bf16 bias (TcScale::bias / TcBlockScale::bias, n bf16 values, null = none).  Then
//   static (scale_c null):  c = fp8(rn(v / s_r)), s_r = *scale_result read on the device, null = 1;
//   dynamic 1 x 128:        d = rn(amax / F) over the row's 128-column block (1 when that is 0, NaN when the block holds
//                           a NaN or an inf), c = fp8(rn(v / d)), d stored at scale_c[i * sc_row + blk * sc_blk].
// fp8() is cvt.rn.satfinite: a finite value past the format's largest F (448, 57344) becomes +-F, NaN stays NaN.
// Their own argument types, so that TcScale and TcBlockScale, and the existing FP8 kernels, keep their layout and code.
struct TcQ8 {
  const float* scale_result;
  float* scale_c;
  long long sc_row, sc_blk;  // element strides of scale_c per row and per 128-column block
  int act;                   // an EpiAct, uniform per launch
};
struct TcScaleQ8 : TcScale { TcQ8 q; };
struct TcBlockScaleQ8 : TcBlockScale { TcQ8 q; };
// Stacked FP8 output (gemm_tc_fp8_q8_stacked_kernel, dynamic 1 x 128 mode only, no bias): the stacked argument plus
// TcQ8 and scale_c's element stride between entries.  Entry e's row i (of the entry) and 128-column block c store
// their scale at scale_c[i_global * sc_row + c * sc_blk] (grouped: i_global the row of the stacked C) or
// scale_c[e * sc_entry_stride + i * sc_row + c * sc_blk] (batch).
struct TcStackScaleQ8 : TcStackScale { TcQ8 q; long long sc_entry_stride; };
struct TcStackBlockScaleQ8 : TcStackBlockScale { TcQ8 q; long long sc_entry_stride; };

// Two fp32 values as two FP8 bytes (lo in the low byte), round to nearest even, finite values saturated.
template <typename OutT>
__device__ __forceinline__ uint32_t cvt_fp8x2(float lo, float hi) {
  uint16_t r;
  if constexpr (std::is_same<OutT, e4m3_out>::value)
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  else
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
// max that returns NaN when either input is NaN (fmaxf drops it): a block's amax carries its NaN
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
// The dynamic scale of a block from its amax: NaN for a NaN or inf amax, else rn(amax / F), 1 when that is 0.
template <typename OutT>
__device__ __forceinline__ float q8_block_scale(float amax) {
  const float d = __fdiv_rn(amax, Fp8Out<OutT>::MAX);
  return !(amax <= 3.402823466e38f) ? __uint_as_float(0x7FC00000u) : d == 0.f ? 1.f : d;
}
// One FP8 pair (col, col + 1) of row `row` into C at byte pitch p.ldc: a 2-byte store where the address allows (any
// base and pitch work).
template <typename OutT>
__device__ __forceinline__ void store_fp8_pair(const TcParams& p, int row, int col, float y0, float y1) {
  const uint32_t w = cvt_fp8x2<OutT>(y0, y1);
  uint8_t* dst = static_cast<uint8_t*>(p.C) + (long long)row * p.ldc + col;
  if (col + 1 < p.N && (reinterpret_cast<uintptr_t>(dst) & 1) == 0) {
    *reinterpret_cast<uint16_t*>(dst) = (uint16_t)w;
  } else {
    dst[0] = (uint8_t)w;
    if (col + 1 < p.N) dst[1] = (uint8_t)(w >> 8);
  }
}

// k == 0 with an FP8 output: v = act(rn(+0 + bias_j)) quantised as fp8_q8_tile does, one thread per row and 128-column
// block, reading no operand and no input scale.
template <typename OutT>
__global__ void fp8_q8_k0_kernel(int m, int n, uint8_t* C, long long ldc, const uint16_t* bias, TcQ8 q) {
  const int qn = (n + 127) / 128;
  const long long items = (long long)m * qn;
  const bool dyn = q.scale_c != nullptr;
  const float sr = !dyn && q.scale_result != nullptr ? *q.scale_result : 1.f;
  TcParams p;
  p.C = C; p.ldc = ldc; p.N = n;
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(it / qn), blk = (int)(it % qn);
    const int c0 = 128 * blk, c1 = min(c0 + 128, n);
    auto val = [&](int j) {
      const float t = __fadd_rn(0.f, bias != nullptr ? __uint_as_float((uint32_t)bias[j] << 16) : -0.f);
      switch (q.act) {
        case ACT_RELU: return epi_act<ACT_RELU>(t);
        case ACT_GELU: return epi_act<ACT_GELU>(t);
        case ACT_GELU_TANH: return epi_act<ACT_GELU_TANH>(t);
        default: return t;
      }
    };
    float amax = 0.f;
    for (int j = c0; j < c1; j++) amax = fmax_nan(amax, fabsf(val(j)));
    const float d = dyn ? q8_block_scale<OutT>(amax) : sr;
    for (int j = c0; j < c1; j += 2)
      store_fp8_pair<OutT>(p, row, j, __fdiv_rn(val(j), d), j + 1 < c1 ? __fdiv_rn(val(j + 1), d) : 0.f);
    if (dyn) q.scale_c[row * q.sc_row + blk * q.sc_blk] = d;
  }
}
// k == 0 of the stacked FP8-output calls: every covered row stores act(rn(+0 + -0)) quantised as fp8_q8_tile does
// (d = 1 for its all-zero blocks) and d.  GROUP: rows [0, end of the last group) of the stacked C, found from the
// clamped offsets (grouped_rows), scales by the row of C.  BATCH: count entries of m rows, C_e = C + e * stride_c,
// scale_c_e = scale_c + e * sc_entry_stride.  One thread per row and 128-column block; no operand, no input scale read.
template <typename OutT, int STACK>
__global__ void fp8_q8_k0_stacked_kernel(const int* __restrict__ offs, int count, int m, int n, uint8_t* C,
                                         long long ldc, long long stride_c, TcQ8 q, long long sc_entry_stride) {
  __shared__ int s_max;
  const int qn = (n + 127) / 128;
  long long rows;
  if constexpr (STACK == STACK_GROUP) rows = grouped_rows(offs, count, m, &s_max);
  else rows = (long long)m * count;
  const long long items = rows * qn;
  TcParams p;
  p.ldc = ldc; p.N = n;
  float v = __fadd_rn(0.f, -0.f);
  switch (q.act) {
    case ACT_RELU: v = epi_act<ACT_RELU>(v); break;
    case ACT_GELU: v = epi_act<ACT_GELU>(v); break;
    case ACT_GELU_TANH: v = epi_act<ACT_GELU_TANH>(v); break;
    default: break;
  }
  const float d = q8_block_scale<OutT>(fabsf(v));
  const float c = __fdiv_rn(v, d);
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += (long long)gridDim.x * blockDim.x) {
    const long long r = it / qn;
    const int blk = (int)(it % qn);
    int row;
    float* sc;
    if constexpr (STACK == STACK_GROUP) {
      row = (int)r;
      p.C = C;
      sc = q.scale_c;
    } else {
      const long long e = r / m;
      row = (int)(r % m);
      p.C = C + e * stride_c;
      sc = q.scale_c + e * sc_entry_stride;
    }
    const int c0 = 128 * blk, c1 = min(c0 + 128, n);
    for (int j = c0; j < c1; j += 2) store_fp8_pair<OutT>(p, row, j, c, j + 1 < c1 ? c : 0.f);
    sc[row * q.sc_row + blk * q.sc_blk] = d;
  }
}
// Shared memory of one stage's block scales: 128 floats of A (one per tile row), then 128 of B (one per tile column).
constexpr int kBlkScaleStageBytes = 2 * 128 * 4;

// The producer warpgroup's scale loaders (BLOCKWISE): warp 1 fills the A half and warp 2 the B half of each stage's
// slot, walking the same tiles and k-blocks as the TMA thread.  Each lane copies its four scales with cp.async and
// has the copies arrive on the stage's full barrier when they land (cp.async.mbarrier.arrive.noinc: 64 arrivals per
// stage), so a loader never waits for a load's latency, only for a free stage, and keeps up with the TMA thread.
// Rows >= M and columns >= N are zero-filled without a read: no load leaves the scale tensors.
constexpr int kBlkScaleArrivals = 2 * 32;
template <class Cfg, int BN, int STAGES>
__device__ __forceinline__ void fp8_block_scale_loader(const TcParams& p, const TcBlockScale& sc, uint32_t slots,
                                                       uint32_t bar_full, uint32_t bar_empty, bool is_b, int lane) {
  // The producer warpgroup runs on 40 registers (setmaxnreg): per tile, one source pointer per lane that advances by
  // the k-block stride, and a step of 32 rows / columns between its four scales (0 for a per-block recipe).
  const float* base = is_b ? sc.b : sc.a;
  const long long blk_stride = is_b ? sc.b_col : sc.a_row, kb_stride = is_b ? sc.b_kb : sc.a_kb;
  const bool per_block = (is_b ? sc.b_blk : sc.a_blk) == 128;
  const int num_kb = (p.K + Cfg::BK - 1) / Cfg::BK;
  const uint32_t half = slots + (is_b ? 512u : 0u) + 4u * lane;
  int s = 0;
  uint32_t ph = 0;
  for (int w = blockIdx.x; w < p.tiles_m * p.tiles_n; w += gridDim.x) {
    int mb, nb;
    tile_coords(w, p.tiles_m, p.tiles_n, p.group_m, mb, nb);
    const int t = is_b ? nb : mb;
    const int i0 = t * (is_b ? BN : Cfg::BM) + lane;
    const int valid = (is_b ? p.N : p.M) - i0;               // scale q of this lane exists iff 32 q < valid
    const float* src = base + (long long)(per_block ? t : i0) * blk_stride;
    const long long step = per_block ? 0 : 32 * blk_stride;
    for (int kb = 0; kb < num_kb; kb++, src += kb_stride) {
      mbar_wait(bar_empty + 8 * s, ph ^ 1);
      const uint32_t dst = half + s * kBlkScaleStageBytes;
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const bool in = 32 * q < valid;
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst + 128u * q), "l"(in ? src + q * step : base),
                     "r"(in ? 4 : 0) : "memory");
      }
      asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar_full + 8 * s) : "memory");
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
}

// The stacked FP8 kernels' group tables (group_table: the clamped ends, then each group's first tile row), static
// shared memory of the GROUPED kernels that read them.
template <int WHICH>
__device__ __forceinline__ int* fp8_group_table() {
  __shared__ int t[kMaxGroups + 1];
  return t;
}

// fp8_block_scale_loader over a stack (TcStackBlockScale): the TMA thread's num_tiles work tiles, each in its entry
// (stack_entry; the group table is built before the warp split).  Per tile one source pointer per lane, at the entry's
// scales: a grouped A's rows are the stacked A's (row end_{e-1} + i), a batch's A and every B start at e * entry
// stride.  A rows >= the entry's M (the next group's, or past the tensor) and B columns >= N are zero-filled without a
// read, so no load leaves the scale tensors whatever the offsets.  A separate function, so that the single-matrix
// loader keeps its code.
template <class Cfg, int BN, int STAGES, int STACK>
__device__ __forceinline__ void fp8_block_scale_loader_stacked(const TcParams& p, const TcStackBlockScale& sc,
                                                               int num_tiles, uint32_t slots, uint32_t bar_full,
                                                               uint32_t bar_empty, bool is_b, int lane) {
  const float* base = is_b ? sc.b : sc.a;
  const long long blk_stride = is_b ? sc.b_col : sc.a_row, kb_stride = is_b ? sc.b_kb : sc.a_kb;
  const bool per_block = (is_b ? sc.b_blk : sc.a_blk) == 128;
  const int num_kb = (p.K + Cfg::BK - 1) / Cfg::BK;
  const uint32_t half = slots + (is_b ? 512u : 0u) + 4u * lane;
  int s = 0;
  uint32_t ph = 0;
  for (int w = blockIdx.x; w < num_tiles; w += gridDim.x) {
    const StackEntry se = stack_entry<STACK>(w, p, sc.st, fp8_group_table<0>(), fp8_group_table<1>());
    int mb, nb;
    tile_coords(w - se.tile0, se.tiles_m, p.tiles_n, p.group_m, mb, nb);
    const int t = is_b ? nb : mb;
    const int i0 = t * (is_b ? BN : Cfg::BM) + lane;
    const int valid = (is_b ? p.N : se.M) - i0;               // scale q of this lane exists iff 32 q < valid
    long long e_off;                                          // elements from base to the entry's first row / column
    if (is_b) e_off = se.entry * sc.b_entry_stride;
    else if constexpr (STACK == STACK_GROUP) e_off = se.a_row * sc.a_row;
    else e_off = se.entry * sc.a_entry_stride;
    const float* src = base + e_off + (long long)(per_block ? t : i0) * blk_stride;
    const long long step = per_block ? 0 : 32 * blk_stride;
    for (int kb = 0; kb < num_kb; kb++, src += kb_stride) {
      mbar_wait(bar_empty + 8 * s, ph ^ 1);
      const uint32_t dst = half + s * kBlkScaleStageBytes;
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const bool in = 32 * q < valid;
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst + 128u * q), "l"(in ? src + q * step : base),
                     "r"(in ? 4 : 0) : "memory");
      }
      asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar_full + 8 * s) : "memory");
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
}
// Work tiles of an FP8 launch: one matrix's, a batch's, or (GROUPED) the table's, built here by every CTA after
// griddep_wait (group_table ends in __syncthreads; CTAs past the table's tiles have no work).
template <int STACK, int BM, class Scale>
__device__ __forceinline__ int fp8_num_tiles(const TcParams& p, const Scale& sc) {
  if constexpr (STACK == STACK_GROUP) {
    group_table(sc.st.offs, sc.st.count, p.M, BM, fp8_group_table<0>(), fp8_group_table<1>());
    return fp8_group_table<1>()[sc.st.count] * p.tiles_n;
  } else if constexpr (STACK == STACK_BATCH) {
    return p.tiles_m * p.tiles_n * sc.st.count;
  } else {
    return p.tiles_m * p.tiles_n;
  }
}

// The GELUs of fp8_q8_tile on the thread's NX values, rolled: each trip applies epi_act to x[0 .. 3] and rotates the
// array by four, so after NX / 4 trips every value has its activation and is back in place.  Fully unrolled (NX
// inlined erfcf / tanhf evaluations), the scheduler's interleaving of the evaluations ran the blockwise kernels out of
// registers; rolled, every FP8-output kernel has 0 spill bytes, at the same time per tile (DESIGN §9).
template <int ACT, int NX>
__device__ __forceinline__ void q8_gelu_rolled(float (&x)[NX]) {
  static_assert(NX % 4 == 0, "groups of four");
#pragma unroll 1
  for (int r = 0; r < NX / 4; r++) {
    float y[4];
#pragma unroll
    for (int i = 0; i < 4; i++) y[i] = epi_act<ACT>(x[i]);
#pragma unroll
    for (int i = 0; i < NX - 4; i++) x[i] = x[i + 4];
#pragma unroll
    for (int i = 0; i < 4; i++) x[NX - 4 + i] = y[i];
  }
}

// The FP8-output store of one consumer thread's part of a tile (TcQ8).  x holds the thread's accumulators (wgmma's
// m64nN layout: x[4j + 2h + e] is row row0 + 8h, column col0 + 8j + e, and the quad of lanes 4r .. 4r + 3 holds all
// columns of its rows), so each 128-column block of a row lies in one quad: j in [16 cb, 16 cb + 16).  Pass 1
// overwrites x with v: the scaling, the bias and ReLU unrolled, the GELUs rolled (q8_gelu_rolled).  Each row-block's
// NaN-carrying amax is then taken over columns < N only; the quad's amax is two shfl.xor steps.  Pass 2 divides,
// converts and stores rows < M and columns < N; lane 4r writes its rows' scales.  The activation is the launch's
// run-time code, tested once per tile: the store is one copy, not one per activation.
template <int BN, typename OutT, bool BLOCKWISE, class Scale, int NX>
__device__ __forceinline__ void fp8_q8_tile(const TcParams& p, const Scale& sc, float (&x)[NX], int row0, int col0,
                                            int lane) {
  constexpr int NB = BN / 128;
  static_assert(BN % 128 == 0 && NX == BN / 2, "whole 128-column blocks per tile");
  const int act = sc.q.act;
  float sa[2] = {0.f, 0.f};
  if constexpr (!BLOCKWISE) {
#pragma unroll
    for (int h = 0; h < 2; h++)
      if (row0 + 8 * h < p.M) sa[h] = __ldg(sc.a + (long long)(row0 + 8 * h) * sc.a_step);
  }
  const unsigned short* bias = static_cast<const unsigned short*>(sc.bias);
#pragma unroll
  for (int j = 0; j < BN / 8; j++) {
    const int col = col0 + 8 * j;
    float sb[2] = {0.f, 0.f}, bi[2] = {-0.f, -0.f};
#pragma unroll
    for (int e = 0; e < 2; e++) {
      if (col + e >= p.N) continue;
      if constexpr (!BLOCKWISE) sb[e] = __ldg(sc.b + (long long)(col + e) * sc.b_step);
      if (bias != nullptr) bi[e] = __uint_as_float((uint32_t)__ldg(bias + col + e) << 16);
    }
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int i = 4 * j + 2 * h + e;
        const float t = __fadd_rn(BLOCKWISE ? x[i] : __fmul_rn(__fmul_rn(x[i], sa[h]), sb[e]), bi[e]);
        x[i] = act == ACT_RELU && t < 0.f ? 0.f : t;                      // epi_act<ACT_RELU>, bit for bit
      }
  }
  if (act == ACT_GELU) q8_gelu_rolled<ACT_GELU>(x);
  else if (act == ACT_GELU_TANH) q8_gelu_rolled<ACT_GELU_TANH>(x);
  float amax[NB][2];
#pragma unroll
  for (int cb = 0; cb < NB; cb++) amax[cb][0] = amax[cb][1] = 0.f;
#pragma unroll
  for (int j = 0; j < BN / 8; j++)
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int e = 0; e < 2; e++)
        if (col0 + 8 * j + e < p.N) amax[j / 16][h] = fmax_nan(amax[j / 16][h], fabsf(x[4 * j + 2 * h + e]));
  const bool dyn = sc.q.scale_c != nullptr;
  float d[NB][2];
  if (dyn) {
#pragma unroll
    for (int cb = 0; cb < NB; cb++)
#pragma unroll
      for (int h = 0; h < 2; h++) {
        float a = amax[cb][h];
        a = fmax_nan(a, __shfl_xor_sync(0xFFFFFFFFu, a, 1));
        a = fmax_nan(a, __shfl_xor_sync(0xFFFFFFFFu, a, 2));
        d[cb][h] = q8_block_scale<OutT>(a);
      }
  } else {
    const float sr = sc.q.scale_result != nullptr ? __ldg(sc.q.scale_result) : 1.f;
#pragma unroll
    for (int cb = 0; cb < NB; cb++) d[cb][0] = d[cb][1] = sr;
  }
#pragma unroll
  for (int j = 0; j < BN / 8; j++)
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int row = row0 + 8 * h, col = col0 + 8 * j;
      if (row >= p.M || col >= p.N) continue;
      const float dd = d[j / 16][h];
      store_fp8_pair<OutT>(p, row, col, __fdiv_rn(x[4 * j + 2 * h], dd), __fdiv_rn(x[4 * j + 2 * h + 1], dd));
    }
  if (dyn && (lane & 3) == 0) {
#pragma unroll
    for (int cb = 0; cb < NB; cb++)
#pragma unroll
      for (int h = 0; h < 2; h++)
        if (row0 + 8 * h < p.M && col0 + 128 * cb < p.N)
          sc.q.scale_c[(long long)(row0 + 8 * h) * sc.q.sc_row + (long long)(col0 / 128 + cb) * sc.q.sc_blk] = d[cb][h];
  }
}

// BLOCKWISE = true: the blockwise-scaled kernels (ProdPromoted, BN = 128, argument TcBlockScale, shared memory
// Cfg::SMEM_BYTES + STAGES * kBlkScaleStageBytes).  The TMA thread and the MMA chain are unchanged; warps 1 and 2 load
// the stage's scales (fp8_block_scale_loader), whose copies also arrive on the stage's full barrier, and each consumer
// warp releases a stage itself (eight arrivals) once its own reads of the stage's scales are done.  false: the code of the
// tensorwise / rowwise kernels, unchanged.
// STACK = STACK_GROUP / STACK_BATCH: the stacked FP8 kernels (argument TcStackScale), gemm_tc_stacked_kernel's schedule
// over this kernel's MMA chains.  Work items are whole tiles, entry outermost (stack_entry); a grouped CTA builds the
// clamped group table after griddep_wait.  A and B are 3-D tensor maps read one entry per box (a grouped A is one
// entry, loaded at row end_g-1 + m0); the store goes through a TcParams whose C and M are the entry's, so rows of a tile
// that belong to the next group are never stored.  Each entry's C is bit for bit the single-matrix kernel's on that
// entry at the same width.  STACK_NONE: the single-matrix kernels, unchanged: every stacked path sits in an
// `if constexpr` branch of its own and the stacking is tested in place (a local constexpr alias for it, like an unused
// local variable, changed the register assignment of those kernels).
// BLOCKWISE with STACK_GROUP / STACK_BATCH (argument TcStackBlockScale): the stacked schedule with the blockwise
// stages; warps 1 and 2 run fp8_block_scale_loader_stacked over the same tiles, and each tile's sum is stored through
// its entry's TcParams with no further scaling and no bias (the single-matrix store's rn(sum + -0) = sum).
// The body is gemm_tc_fp8_body, shared with gemm_tc_fp8_q8_stacked_kernel (below), the stacked FP8-output kernels.
// Its parameters are taken by value: with references the tensorwise / rowwise kernels' register assignment changed.
template <int KIND, int BN, int STAGES, typename OutT, class Prod, bool BLOCKWISE, int STACK, class Scale>
__device__ __forceinline__ void gemm_tc_fp8_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcParams p,
                                                 const Scale sc) {
  using Cfg = TcConfig<KIND, BN, STAGES, Prod, 128>;
  using MMA = typename Cfg::MMA;
  static_assert(KIND == KIND_E4M3 || KIND == KIND_E4M3E5M2 || KIND == KIND_E5M2E4M3, "FP8 kinds");
  static_assert(!Cfg::A_MN && !Cfg::B_MN && Prod::NPA == 1 && Prod::NPB == 1, "FP8: K-major A and B, one plane");
  static_assert(std::is_same<OutT, float>::value || OutBytes<OutT>::V == 2 || Fp8Out<OutT>::V, "FP8: fp32, 16-bit or FP8 C");
  static_assert(!Fp8Out<OutT>::V || BN % 128 == 0, "FP8 C: tiles of whole 128-column scale blocks");
  static_assert(!BLOCKWISE || (std::is_same<Prod, ProdPromoted>::value && BN == 128 && Cfg::BK == 128),
                "blockwise scales: one 128-element k-block per promotion, tiles on the 128 x 128 scale blocks");
  static_assert(!BLOCKWISE || Cfg::SMEM_BYTES + STAGES * kBlkScaleStageBytes <= 232448, "blockwise: shared memory");
  static_assert(!(BLOCKWISE && STACK == STACK_GROUP) ||
                    Cfg::SMEM_BYTES + STAGES * kBlkScaleStageBytes + 2 * (kMaxGroups + 1) * (int)sizeof(int) <= 232448,
                "grouped blockwise: the pipeline, the scale slots and the group tables exceed 227 KB of shared memory");
  static_assert(STACK == STACK_NONE || STACK == STACK_GROUP || STACK == STACK_BATCH, "stacked FP8: a batch or a grouped call");
  static_assert(STACK != STACK_GROUP || Cfg::SMEM_BYTES + 2 * (kMaxGroups + 1) * (int)sizeof(int) <= 232448,
                "the pipeline and the group tables exceed the 227 KB of shared memory of sm_90");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // swizzle atoms need 1 KB
  const uint32_t sA = smem_base;
  const uint32_t sB = sA + STAGES * Cfg::A_STAGE;
  const uint32_t bar_full = sB + STAGES * Cfg::B_STAGE;
  const uint32_t bar_empty = bar_full + 8 * STAGES;
  [[maybe_unused]] const uint32_t s_scale = bar_empty + 8 * STAGES;   // BLOCKWISE: STAGES slots of kBlkScaleStageBytes

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; i++) {
      mbar_init(bar_full + 8 * i, BLOCKWISE ? 1 + kBlkScaleArrivals : 1);
      mbar_init(bar_empty + 8 * i, BLOCKWISE ? Cfg::EPI_WARPS : Cfg::CONSUMERS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_launch();
  griddep_wait();

  const int num_tiles = fp8_num_tiles<STACK, Cfg::BM>(p, sc);   // STACK_GROUP: builds the group table first
  const int num_kb = (p.K + Cfg::BK - 1) / Cfg::BK;

  if (warp < 4) {
    // ===================== TMA producer (warpgroup 0) =====================
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      if constexpr (STACK != STACK_NONE) {                       // one entry per 3-D box; a grouped A at row end_{g-1} + m0
        for (int w = blockIdx.x; w < num_tiles; w += gridDim.x) {
          const StackEntry se = stack_entry<STACK>(w, p, sc.st, fp8_group_table<0>(), fp8_group_table<1>());
          int mb, nb;
          tile_coords(w - se.tile0, se.tiles_m, p.tiles_n, p.group_m, mb, nb);
          const int m0 = se.a_row + mb * Cfg::BM, n0 = nb * BN;
          for (int kb = 0; kb < num_kb; kb++) {
            mbar_wait(bar_empty + 8 * s, ph ^ 1);
            const uint32_t full = bar_full + 8 * s;
            mbar_arrive_expect_tx(full, Cfg::STAGE_BYTES);
            tma_load_3d(sA + s * Cfg::A_STAGE, &tmA, full, kb * Cfg::BK, m0, se.a_entry);
            tma_load_3d(sB + s * Cfg::B_STAGE, &tmB, full, kb * Cfg::BK, n0, se.b_entry);
            if (++s == STAGES) { s = 0; ph ^= 1; }
          }
        }
      } else {
        for (int w = blockIdx.x; w < num_tiles; w += gridDim.x) {
          int mb, nb;
          tile_coords(w, p.tiles_m, p.tiles_n, p.group_m, mb, nb);
          const int m0 = mb * Cfg::BM, n0 = nb * BN;
          for (int kb = 0; kb < num_kb; kb++) {
            mbar_wait(bar_empty + 8 * s, ph ^ 1);
            const uint32_t full = bar_full + 8 * s;
            mbar_arrive_expect_tx(full, Cfg::STAGE_BYTES);
            tma_load_2d(sA + s * Cfg::A_STAGE, &tmA, full, kb * Cfg::BK, m0);
            tma_load_2d(sB + s * Cfg::B_STAGE, &tmB, full, kb * Cfg::BK, n0);
            if (++s == STAGES) { s = 0; ph ^= 1; }
          }
        }
      }
    }
    if constexpr (BLOCKWISE && STACK != STACK_NONE) {
      if (warp == 1 || warp == 2)
        fp8_block_scale_loader_stacked<Cfg, BN, STAGES, STACK>(p, sc, num_tiles, s_scale, bar_full, bar_empty, warp == 2,
                                                               lane);
    } else if constexpr (BLOCKWISE) {
      if (warp == 1 || warp == 2)
        fp8_block_scale_loader<Cfg, BN, STAGES>(p, sc, s_scale, bar_full, bar_empty, warp == 2, lane);
    }
  } else {
    // ===================== consumers (warpgroups 1 and 2): MMA chain + scaled epilogue =====================
    setmaxnreg_inc<232>();
    const int cw = warp / 4 - 1;
    const int ew = warp - 4;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    int s = 0;
    uint32_t ph = 0;
    float acc[Cfg::ACC];
    float sum[Cfg::REGACC ? Cfg::ACC : 1];
    // BLOCKWISE: this thread's rows and first column inside the tile, and its A scales of the current k-block (and B's,
    // when b_blk = 128: one value for the tile), read from the stage's slot before the MMAs are issued.
    [[maybe_unused]] const int r_loc = ew * 16 + (lane >> 2), c_loc = 2 * (lane & 3);
    [[maybe_unused]] float ssa[2] = {0.f, 0.f}, ssb = 0.f;
    for (int w = blockIdx.x; w < num_tiles; w += gridDim.x) {
      int mb, nb;
      if constexpr (STACK != STACK_NONE) {
        const StackEntry se = stack_entry<STACK>(w, p, sc.st, fp8_group_table<0>(), fp8_group_table<1>());
        tile_coords(w - se.tile0, se.tiles_m, p.tiles_n, p.group_m, mb, nb);
      } else {
        tile_coords(w, p.tiles_m, p.tiles_n, p.group_m, mb, nb);
      }
      const int m0 = mb * Cfg::BM, n0 = nb * BN;      // stacked: m0 is a row inside the entry
      const int chunk = BLOCKWISE ? 1 : Cfg::REGACC ? p.chunk_kb : num_kb;
      for (int c0 = 0; c0 < num_kb; c0 += chunk) {
        const int c1 = min(c0 + chunk, num_kb);
        int prev = -1;
        for (int kb = c0; kb < c1; kb++) {
          mbar_wait(bar_full + 8 * s, ph);
          if constexpr (BLOCKWISE) {
            const float* slot = reinterpret_cast<const float*>(smem_raw + (s_scale - smem_u32(smem_raw))) +
                                s * (kBlkScaleStageBytes / 4);
            ssa[0] = slot[r_loc];
            ssa[1] = slot[r_loc + 8];
            if (sc.b_blk == 128) ssb = slot[128];
          }
          const uint32_t a0 = sA + s * Cfg::A_STAGE + cw * Cfg::A_WG;
          const uint32_t b0 = sB + s * Cfg::B_STAGE;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < Cfg::MMAS_PER_STAGE; k++) {
            const uint64_t ad = make_sdesc(a0 + k * Cfg::A_KADV, 16, Cfg::A_SBO, Cfg::A_SWZ);
            const uint64_t bd = make_sdesc(b0 + k * Cfg::B_KADV, 16, Cfg::A_SBO, Cfg::A_SWZ);
            MMA::mma(acc, ad, bd, ((kb - c0) | k) != 0 ? 1u : 0u);
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (!BLOCKWISE && prev >= 0 && wg_leader) mbar_arrive(bar_empty + 8 * prev);
          prev = s;
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if constexpr (BLOCKWISE) {
          // sum = fma(acc, rn(sa * sb), sum), from sum = +0; then this warp's reads of the stage are done and it
          // releases the stage (one arrival per consumer warp)
          if (sc.b_blk == 128) {
            const float s2[2] = {__fmul_rn(ssa[0], ssb), __fmul_rn(ssa[1], ssb)};
#pragma unroll
            for (int i = 0; i < Cfg::ACC; i++) sum[i] = __fmaf_rn(acc[i], s2[(i >> 1) & 1], c0 == 0 ? 0.f : sum[i]);
          } else {
            const float* slot = reinterpret_cast<const float*>(smem_raw + (s_scale - smem_u32(smem_raw))) +
                                prev * (kBlkScaleStageBytes / 4) + 128 + c_loc;
#pragma unroll
            for (int j = 0; j < BN / 8; j++) {
              const float2 b2 = *reinterpret_cast<const float2*>(slot + 8 * j);
#pragma unroll
              for (int i = 4 * j; i < 4 * j + 4; i++)
                sum[i] = __fmaf_rn(acc[i], __fmul_rn(ssa[(i >> 1) & 1], i & 1 ? b2.y : b2.x), c0 == 0 ? 0.f : sum[i]);
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
        } else {
          if (prev >= 0 && wg_leader) mbar_arrive(bar_empty + 8 * prev);
          if constexpr (Cfg::REGACC) {
#pragma unroll
            for (int i = 0; i < Cfg::ACC; i++) sum[i] = c0 == 0 ? acc[i] : __fadd_rn(sum[i], acc[i]);
          }
        }
      }

      // ---- this warp's 16 rows of the tile into C: (acc * sa) * sb (BLOCKWISE: sum), then + bias in store_pair ----
      const int row0 = m0 + ew * 16 + (lane >> 2);
      const int col0 = n0 + 2 * (lane & 3);
      if constexpr (Fp8Out<OutT>::V && STACK != STACK_NONE) {
        // stacked FP8 C (TcStackScaleQ8 / TcStackBlockScaleQ8): the entry's C and rows, and its scales as a
        // single-matrix argument (B's at its entry, no bias), then fp8_q8_tile stores exactly what the single-matrix
        // kernel stores for that entry.  A group is rows [a_row, a_row + M) of the stacked C, of A's scales and of
        // scale_c, all indexed by that row: its tile rows are shifted by a_row and masked at the group's end (fewer live
        // registers than rebased pointers, which spilled at BN = 256).  A batch entry's C, A scales and scale_c start
        // at its entry strides.
        const StackEntry se = stack_entry<STACK>(w, p, sc.st, fp8_group_table<0>(), fp8_group_table<1>());
        TcParams pc = p;
        typename std::conditional<BLOCKWISE, TcBlockScaleQ8, TcScaleQ8>::type ve;
        static_cast<typename std::conditional<BLOCKWISE, TcBlockScale, TcScale>::type&>(ve) = sc;
        ve.b = sc.b + se.entry * sc.b_entry_stride;
        ve.bias = nullptr;
        ve.q = sc.q;
        int r0 = row0;
        if constexpr (STACK == STACK_GROUP) {
          pc.M = se.a_row + se.M;
          r0 += se.a_row;
        } else {
          pc.C = static_cast<uint8_t*>(p.C) + se.c_off;
          pc.M = se.M;
          ve.a = sc.a + se.entry * sc.a_entry_stride;
          ve.q.scale_c = sc.q.scale_c + se.entry * sc.sc_entry_stride;
        }
        if constexpr (Cfg::REGACC) fp8_q8_tile<BN, OutT, BLOCKWISE>(pc, ve, sum, r0, col0, lane);
        else fp8_q8_tile<BN, OutT, BLOCKWISE>(pc, ve, acc, r0, col0, lane);
        continue;
      } else if constexpr (Fp8Out<OutT>::V) {
        // FP8 C (TcQ8): v, then the static or dynamic quantisation, in fp8_q8_tile
        if constexpr (Cfg::REGACC) fp8_q8_tile<BN, OutT, BLOCKWISE>(p, sc, sum, row0, col0, lane);
        else fp8_q8_tile<BN, OutT, BLOCKWISE>(p, sc, acc, row0, col0, lane);
        continue;
      }
      if constexpr (BLOCKWISE && STACK != STACK_NONE) {
        // the entry's C and rows, as below; the blockwise sum is stored as is (no bias)
        const StackEntry se = stack_entry<STACK>(w, p, sc.st, fp8_group_table<0>(), fp8_group_table<1>());
        TcParams pc = p;
        pc.C = static_cast<uint8_t*>(p.C) + se.c_off * OutBytes<OutT>::V;
        pc.M = se.M;
        const int ce[2] = {0, 0};
#pragma unroll
        for (int j = 0; j < BN / 8; j++)
#pragma unroll
          for (int h = 0; h < 2; h++)
            store_pair<OutT, float, ACT_NONE>(pc, row0 + 8 * h, col0 + 8 * j, sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1],
                                              false, false, 1.f, 1.f, 0, ce, 0.f, 0.f);
        continue;
      }
      if constexpr (STACK != STACK_NONE && !BLOCKWISE) {
        // the entry's C and rows (pc; rows of the tile past the entry's are never stored), and its scale vectors: row i
        // of the entry takes sa_e[i], column j sb_e[j].  No bias.  (A copy of the store below, so that the
        // single-matrix kernels keep their code.)
        const StackEntry se = stack_entry<STACK>(w, p, sc.st, fp8_group_table<0>(), fp8_group_table<1>());
        TcParams pc = p;
        pc.C = static_cast<uint8_t*>(p.C) + se.c_off * OutBytes<OutT>::V;
        pc.M = se.M;
        const float* sa_e = sc.a + (STACK == STACK_GROUP ? (long long)se.a_row : se.entry * sc.a_entry_stride);
        const float* sb_e = sc.b + se.entry * sc.b_entry_stride;
        float sa[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; h++)
          if (row0 + 8 * h < pc.M) sa[h] = __ldg(sa_e + row0 + 8 * h);
        const int ce[2] = {0, 0};
#pragma unroll
        for (int j = 0; j < BN / 8; j++) {
          const int col = col0 + 8 * j;
          float sb[2] = {0.f, 0.f};
#pragma unroll
          for (int e = 0; e < 2; e++)
            if (col + e < p.N) sb[e] = __ldg(sb_e + col + e);
#pragma unroll
          for (int h = 0; h < 2; h++) {
            const float v0 = Cfg::REGACC ? sum[4 * j + 2 * h] : acc[4 * j + 2 * h];
            const float v1 = Cfg::REGACC ? sum[4 * j + 2 * h + 1] : acc[4 * j + 2 * h + 1];
            store_pair<OutT, float, ACT_NONE>(pc, row0 + 8 * h, col, __fmul_rn(__fmul_rn(v0, sa[h]), sb[0]),
                                              __fmul_rn(__fmul_rn(v1, sa[h]), sb[1]), false, false, 1.f, 1.f, 0, ce, 0.f,
                                              0.f);
          }
        }
        continue;
      }
      float sa[2] = {0.f, 0.f};
      if constexpr (!BLOCKWISE) {
#pragma unroll
        for (int h = 0; h < 2; h++)
          if (row0 + 8 * h < p.M) sa[h] = __ldg(sc.a + (long long)(row0 + 8 * h) * sc.a_step);
      }
      const int ce[2] = {0, 0};
#pragma unroll
      for (int j = 0; j < BN / 8; j++) {
        const int col = col0 + 8 * j;
        float sb[2] = {0.f, 0.f}, bi[2] = {-0.f, -0.f};
#pragma unroll
        for (int e = 0; e < 2; e++) {
          if (col + e >= p.N) continue;
          if constexpr (!BLOCKWISE) sb[e] = __ldg(sc.b + (long long)(col + e) * sc.b_step);
          if (sc.bias != nullptr) {
            if constexpr (std::is_same<OutT, float>::value)
              bi[e] = __ldg(reinterpret_cast<const float*>(sc.bias) + col + e);
            else
              bi[e] = c16_to_f32<OutT>(__ldg(reinterpret_cast<const unsigned short*>(sc.bias) + col + e));
          }
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const float v0 = Cfg::REGACC ? sum[4 * j + 2 * h] : acc[4 * j + 2 * h];
          const float v1 = Cfg::REGACC ? sum[4 * j + 2 * h + 1] : acc[4 * j + 2 * h + 1];
          if constexpr (BLOCKWISE)
            store_pair<OutT, float, ACT_NONE>(p, row0 + 8 * h, col, v0, v1, false, false, 1.f, 1.f, 0, ce, 0.f, 0.f, bi[0],
                                              bi[1]);
          else
            store_pair<OutT, float, ACT_NONE>(p, row0 + 8 * h, col, __fmul_rn(__fmul_rn(v0, sa[h]), sb[0]),
                                              __fmul_rn(__fmul_rn(v1, sa[h]), sb[1]), false, false, 1.f, 1.f, 0, ce, 0.f,
                                              0.f, bi[0], bi[1]);
        }
      }
    }
  }
}

template <int KIND, int BN, int STAGES, typename OutT, class Prod, bool BLOCKWISE = false, int STACK = STACK_NONE>
__global__ void __launch_bounds__((TcConfig<KIND, BN, STAGES, Prod, 128>::THREADS), 1)
gemm_tc_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcParams p,
                   const typename std::conditional<
                       Fp8Out<OutT>::V, typename std::conditional<BLOCKWISE, TcBlockScaleQ8, TcScaleQ8>::type,
                       typename std::conditional<
                           BLOCKWISE, typename std::conditional<STACK != STACK_NONE, TcStackBlockScale, TcBlockScale>::type,
                           typename std::conditional<STACK != STACK_NONE, TcStackScale, TcScale>::type>::type>::type sc) {
  static_assert(!Fp8Out<OutT>::V || STACK == STACK_NONE, "stacked FP8 C: gemm_tc_fp8_q8_stacked_kernel");
  gemm_tc_fp8_body<KIND, BN, STAGES, OutT, Prod, BLOCKWISE, STACK>(tmA, tmB, p, sc);
}

// The stacked FP8-output kernels (STACK_GROUP / STACK_BATCH, OutT e4m3_out / e5m2_out, dynamic 1 x 128 mode): every
// entry's C and scale_c are the single-matrix FP8-output kernel's on that entry at the same width.  A __global__ of
// their own over the same body, so that gemm_tc_fp8_kernel's instantiations stay the FP8 kernels with an fp32 or
// 16-bit C, or one FP8 C matrix.
template <int KIND, int BN, int STAGES, typename OutT, class Prod, bool BLOCKWISE, int STACK>
__global__ void __launch_bounds__((TcConfig<KIND, BN, STAGES, Prod, 128>::THREADS), 1)
gemm_tc_fp8_q8_stacked_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                              const TcParams p,
                              const typename std::conditional<BLOCKWISE, TcStackBlockScaleQ8, TcStackScaleQ8>::type sc) {
  static_assert(Fp8Out<OutT>::V && STACK != STACK_NONE, "stacked FP8 C");
  gemm_tc_fp8_body<KIND, BN, STAGES, OutT, Prod, BLOCKWISE, STACK>(tmA, tmB, p, sc);
}

// ---- stacked 16-bit GEMMs: strided batch and grouped (torch._grouped_mm) --------------------------------------------
// gemm_tc_kernel's persistent schedule over a stack of matrices, cut down to what the stacked calls need: 16-bit
// operands, one plane, 128-byte rows, fp32 or 16-bit C, no bias / activation, no scaling.  It is a kernel of its own
// rather than a flag of gemm_tc_kernel so that the single-matrix kernels keep their code exactly.  Its MMA chain
// (k-blocks in order, one accumulator) and its epilogue (store_pair, the same fold / alpha / beta rules) are
// gemm_tc_kernel's, so every entry equals the single-matrix call on that entry bit for bit at the same tile width.
// Work item w covers the tiles of every entry, entry outermost: one entry's tiles are adjacent and share its B in L2;
// inside an entry tile_coords walks its raster groups as for one matrix.  A and B are 3-D tensor maps (inner, rows,
// entry) read one entry per box, so TMA's zero fill past the rows and the inner extent stays inside the entry.
//   Strided batch: entry e is A_e, B_e and C + e * stride_c (64-bit), tiles_m x tiles_n tiles each.  The K-split tail
//   (fp32 C) cuts the last partial round of the whole batch.
//   GROUPED: group g is rows [end_g-1, end_g) of one stacked row-major A (total_m = p.M rows) and C, times B_g, entry g
//   of B.  The group sizes exist only on the device, so the schedule is built here: after griddep_wait every CTA reads
//   the offsets, clamps them and scans the 128-row tiles of each group into shared memory (group_table); producer and
//   consumers find a tile's group by binary search.  A is one entry: a tile at row end_g-1 + 128 mb may load rows of
//   the next group (or TMA's zeros past total_m), but each row of C depends only on its own row of A, and store_pair,
//   on a TcParams whose C starts at row end_g-1 and whose M is the group's rows, never stores those rows.  The host
//   sizes the grid for a bound on the tiles (p.tiles_m tile rows) and takes no K split (split = 1, full_tiles = that
//   bound): it does not know the tile count.
//   KGROUP (the weight gradient of a grouped layer, torch._grouped_mm 2-D x 2-D): group g is K rows
//   [end_g-1, end_g) of one A^T (total_k x m, p.K = total_k) and one B (total_k x n), both MN-major and read as one
//   entry; C_g = C + g * stride_c is a whole m x n matrix.  The tiles are a batch's (entry outermost, p.tiles_m x
//   p.tiles_n per group, known to the host), whole tiles only.  Every CTA builds the clamped K ends (group_table) after
//   griddep_wait.  k-block kb of group g is loaded at K row end_g-1 + 64 kb; the last one of a group whose k_g is not a
//   multiple of 64 also holds rows of the next group (real data: 0 * inf would be NaN) or TMA's zeros past total_k, so
//   the consumers zero its rows >= k_g - 64 kb in shared memory before its MMAs (zero_k_tail).  The MMA count is
//   unchanged, so every C_g is bit for bit the _ex call with k = k_g, whose TMA zero-fills those rows.  A group with
//   k_g = 0 issues no loads or MMAs and stores the _ex k == 0 result (store_beta_c).
// StackEntry / stack_entry (above gemm_tc_fp8_kernel, which shares them) find a work tile's entry.

// KGROUP: zeroes K rows [r0, BK) of one stage's MN-major boxes (A's, then B's; contiguous in shared memory), where one
// K row of a SWIZZLE_128B box is one whole 128-byte line, so no swizzle arithmetic is needed.  The 256 consumer threads
// share the lines; each then makes its stores visible to the tensor cores' async proxy, and both consumer warpgroups
// meet at named barrier 1 before either issues the stage's MMAs.
template <class Cfg>
__device__ __forceinline__ void zero_k_tail(uint32_t sA_stage, uint32_t sB_stage, int r0, int tid) {
  static_assert(Cfg::A_MN && Cfg::B_MN, "K-grouped: MN-major A and B");
  constexpr int BOXES = Cfg::A_BOXES + Cfg::B_BOXES;
  static_assert(Cfg::A_STAGE == Cfg::A_BOXES * Cfg::MN_BOX_BYTES && Cfg::B_BOX_BYTES == Cfg::MN_BOX_BYTES,
                "K-grouped: the stage is A's boxes then B's, each BK lines of 128 bytes");
  const int rows = Cfg::BK - r0;
  const int chunks = BOXES * rows * 8;                              // 16-byte chunks to clear
  for (int i = tid; i < chunks; i += 256) {
    const int box = i / (rows * 8), rest = i - box * (rows * 8);
    const int line = r0 + (rest >> 3);
    const uint32_t base = box < Cfg::A_BOXES ? sA_stage + box * Cfg::MN_BOX_BYTES
                                             : sB_stage + (box - Cfg::A_BOXES) * Cfg::MN_BOX_BYTES;
    const uint32_t addr = base + line * 128 + (rest & 7) * 16;
    asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(addr), "r"(0u) : "memory");
  }
  fence_proxy_async();
  asm volatile("bar.sync 1, 256;" ::: "memory");
}

// KGROUP, a group with k_g = 0: the element of the _ex call with k == 0, round_out(beta * float(C)), or raw +0 without
// reading C when beta == 0 (not fma(beta, C, alpha * 0), whose zero signs differ).
template <typename OutT>
__device__ __forceinline__ void store_beta_c(const TcParams& p, int row, int col, float be) {
  if (row >= p.M || col >= p.N) return;
  if constexpr (std::is_same<OutT, float>::value) {
    float* dst = reinterpret_cast<float*>(p.C) + (long long)row * p.ldc + col;
    *dst = be != 0.f ? be * *dst : 0.f;
  } else {
    uint16_t* dst = reinterpret_cast<uint16_t*>(p.C) + (long long)row * p.ldc + col;
    if (be == 0.f) { *dst = 0; return; }
    const float x = be * c16_to_f32<OutT>(*dst);
    const uint32_t w = std::is_same<OutT, f16_out>::value ? cvt_f16x2(x, 0.f) : cvt_bf16x2(x, 0.f);
    *dst = (uint16_t)w;
  }
}

template <int KIND, int BN, int STAGES, typename OutT, int AL, int BL, int STACK>
__global__ void __launch_bounds__((TcConfig<KIND, BN, STAGES, ProdSingle, 128, AL, BL>::THREADS), 1)
gemm_tc_stacked_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const TcParams p, const TcStack st) {
  using Cfg = TcConfig<KIND, BN, STAGES, ProdSingle, 128, AL, BL>;
  using MMA = typename Cfg::MMA;
  using Acc = typename MMA::Acc;
  constexpr bool GROUPED = STACK == STACK_GROUP, KGROUP = STACK == STACK_KGROUP;
  static_assert(KindTraits<KIND>::ELEM == 2 && (std::is_same<OutT, float>::value || OutBytes<OutT>::V == 2),
                "stacked: 16-bit kinds with fp32 or 16-bit C");
  static_assert(STACK == STACK_BATCH || GROUPED || KGROUP, "stacked: a batch, a grouped or a K-grouped call");
  static_assert(!GROUPED || AL == LAYOUT_K, "grouped: A is row-major");
  static_assert(!KGROUP || (AL == LAYOUT_MN && BL == LAYOUT_MN), "K-grouped: A^T and B, both MN-major");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // swizzle atoms need 1 KB
  const uint32_t sA = smem_base;
  const uint32_t sB = sA + STAGES * Cfg::A_STAGE;
  const uint32_t bar_full = sB + STAGES * Cfg::B_STAGE;
  const uint32_t bar_empty = bar_full + 8 * STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; i++) {
      mbar_init(bar_full + 8 * i, 1);
      mbar_init(bar_empty + 8 * i, Cfg::CONSUMERS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  griddep_launch();
  griddep_wait();

  const int* grp_end = nullptr;               // GROUPED: group g is rows [grp_end[g], grp_end[g + 1])
  const int* grp_tile = nullptr;              //          and tiles [grp_tile[g], grp_tile[g + 1]) of the tile order
  int num_tiles;                              // KGROUP: group g is K rows [grp_end[g], grp_end[g + 1])
  if constexpr (GROUPED || KGROUP) {          // the batched kernels declare no tables
    static_assert(Cfg::SMEM_BYTES + 2 * (kMaxGroups + 1) * (int)sizeof(int) <= 232448,
                  "the pipeline and the group tables exceed the 227 KB of shared memory of sm_90");
    __shared__ int s_end[kMaxGroups + 1];
    __shared__ int s_tile[kMaxGroups + 1];
    if constexpr (GROUPED) {
      group_table(st.offs, st.count, p.M, Cfg::BM, s_end, s_tile);   // ends in __syncthreads
      grp_end = s_end;
      grp_tile = s_tile;
      num_tiles = grp_tile[st.count] * p.tiles_n;                    // CTAs past it have no work
    } else {
      group_table(st.offs, st.count, p.K, Cfg::BK, s_end, s_tile);   // only the K ends are used
      grp_end = s_end;
      num_tiles = p.tiles_m * p.tiles_n * st.count;
    }
  } else {
    num_tiles = p.tiles_m * p.tiles_n * st.count;
  }
  const int num_items = p.full_tiles + (num_tiles - p.full_tiles) * p.split;
  const int num_kb = (p.K + Cfg::BK - 1) / Cfg::BK;
  // GROUPED and KGROUP work items are whole tiles (split = 1), known at compile time: with a run-time part the split
  // tail's branches stay in the epilogue, and ptxas specialises its store loop less (DESIGN §9: 1-2.5 % slower on an
  // H100).  A KGROUP tile's k-blocks are its group's.

  if (warp < 4) {
    // ===================== TMA producer (warpgroup 0) =====================
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int w = blockIdx.x; w < num_items; w += gridDim.x) {
        WorkItem it = STACK == STACK_BATCH ? work_item(w, p, num_kb) : WorkItem{w, 0, 0, num_kb};
        const StackEntry se = stack_entry<STACK>(it.tile, p, st, grp_end, grp_tile);
        if constexpr (KGROUP) it.kb1 = (se.k_len + Cfg::BK - 1) / Cfg::BK;
        int mb, nb;
        tile_coords(it.tile - se.tile0, se.tiles_m, p.tiles_n, p.group_m, mb, nb);
        const int m0 = se.a_row + mb * Cfg::BM, n0 = nb * BN;
        for (int kb = it.kb0; kb < it.kb1; kb++) {
          mbar_wait(bar_empty + 8 * s, ph ^ 1);
          const uint32_t full = bar_full + 8 * s;
          mbar_arrive_expect_tx(full, Cfg::STAGE_BYTES);
          const int kr = se.k0 + kb * Cfg::BK;        // K row of the box (se.k0 = 0 but for KGROUP)
          if constexpr (Cfg::A_MN) {                  // A^T (k x m): one 64-column box per consumer
#pragma unroll
            for (int j = 0; j < Cfg::A_BOXES; j++)
              tma_load_3d(sA + s * Cfg::A_STAGE + j * Cfg::MN_BOX_BYTES, &tmA, full, m0 + j * Cfg::MN_BOX_COLS,
                          kr, se.a_entry);
          } else {
            tma_load_3d(sA + s * Cfg::A_STAGE, &tmA, full, kr, m0, se.a_entry);
          }
          if constexpr (!Cfg::B_MN) {                 // B^T (n x k): one box of BN rows
            tma_load_3d(sB + s * Cfg::B_STAGE, &tmB, full, kr, n0, se.b_entry);
          } else {
#pragma unroll
            for (int j = 0; j < Cfg::B_BOXES; j++)
              tma_load_3d(sB + s * Cfg::B_STAGE + j * Cfg::B_BOX_BYTES, &tmB, full, n0 + j * Cfg::B_BOX_COLS,
                          kr, se.b_entry);
          }
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers (warpgroups 1 and 2): MMA chain + epilogue =====================
    setmaxnreg_inc<232>();
    const int cw = warp / 4 - 1;                    // consumer warpgroup: rows [64 cw, 64 cw + 64) of the tile
    const int ew = warp - 4;                        // consumer warp 0..7: 16 rows each
    const bool wg_leader = (threadIdx.x & 127) == 0;
    const uint32_t b_lbo = p.dbg_b_lbo ? (uint32_t)p.dbg_b_lbo : (uint32_t)Cfg::B_BOX_BYTES;
    const uint32_t b_sbo = p.dbg_b_sbo ? (uint32_t)p.dbg_b_sbo : 1024u;
    int s = 0;
    uint32_t ph = 0;
    Acc acc[Cfg::ACC];
    for (int w = blockIdx.x; w < num_items; w += gridDim.x) {
      WorkItem it = STACK == STACK_BATCH ? work_item(w, p, num_kb) : WorkItem{w, 0, 0, num_kb};
      const StackEntry se = stack_entry<STACK>(it.tile, p, st, grp_end, grp_tile);
      if constexpr (KGROUP) it.kb1 = (se.k_len + Cfg::BK - 1) / Cfg::BK;
      int mb, nb;
      tile_coords(it.tile - se.tile0, se.tiles_m, p.tiles_n, p.group_m, mb, nb);
      const int m0 = mb * Cfg::BM, n0 = nb * BN;      // m0: row inside the entry
      int prev = -1;
      for (int kb = it.kb0; kb < it.kb1; kb++) {
        mbar_wait(bar_full + 8 * s, ph);
        const uint32_t a0 = sA + s * Cfg::A_STAGE + cw * Cfg::A_WG;
        const uint32_t b0 = sB + s * Cfg::B_STAGE;
        if constexpr (KGROUP) {                        // the group's last box: rows past k_g are not its own
          const int r0 = se.k_len - kb * Cfg::BK;
          if (r0 < Cfg::BK) zero_k_tail<Cfg>(sA + s * Cfg::A_STAGE, b0, r0, threadIdx.x - 128);
        }
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < Cfg::MMAS_PER_STAGE; k++) {
          uint64_t ad, bd;
          if constexpr (Cfg::A_MN) ad = make_sdesc(a0 + k * Cfg::A_KADV, Cfg::MN_BOX_BYTES, 1024, SWZ_128B);
          else ad = make_sdesc(a0 + k * Cfg::A_KADV, 16, Cfg::A_SBO, Cfg::A_SWZ);
          if constexpr (Cfg::B_MN) bd = make_sdesc(b0 + k * Cfg::B_KADV, b_lbo, b_sbo, SWZ_128B);
          else bd = make_sdesc(b0 + k * Cfg::B_KADV, 16, Cfg::A_SBO, Cfg::A_SWZ);
          MMA::mma(acc, ad, bd, ((kb - it.kb0) | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();                              // the previous k-block's products retired: its stage is free
        if (prev >= 0 && wg_leader) mbar_arrive(bar_empty + 8 * prev);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && wg_leader) mbar_arrive(bar_empty + 8 * prev);

      // ---- this warp's 16 rows of the tile into the entry's C ----
      int* flag = p.flags + (it.tile - p.full_tiles) * Cfg::EPI_WARPS + ew;
      if (it.part > 0) {                               // K-split tail: wait until parts < it.part are in C
        if (lane == 0) {
          const long long t0 = clock64();
          while (true) {
            int v;
            asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
            if (v == it.part) break;
            if (clock64() - t0 > 4000000000LL) { asm volatile("trap;"); }
          }
        }
        __syncwarp();
      }
      const bool fold = p.accumulate != 0 || it.part > 0 || (p.axpby && p.beta != 0.f);
      const float al = p.axpby ? p.alpha : 1.f;
      const float be = (p.axpby && it.part == 0) ? p.beta : 1.f;
      const int row0 = m0 + ew * 16 + (lane >> 2);
      const int col0 = n0 + 2 * (lane & 3);
      TcParams pc = p;
      pc.C = static_cast<uint8_t*>(p.C) + se.c_off * OutBytes<OutT>::V;
      pc.M = se.M;
      if constexpr (KGROUP) {
        if (it.kb1 == 0) {                             // an empty group: the _ex k == 0 result
          const float beta0 = p.axpby ? p.beta : 0.f;
          for (int j = 0; j < BN / 8; j++)
            for (int h = 0; h < 2; h++)
              for (int e = 0; e < 2; e++) store_beta_c<OutT>(pc, row0 + 8 * h, col0 + 8 * j + e, beta0);
          continue;
        }
      }
      const int ce[2] = {0, 0};
#pragma unroll
      for (int j = 0; j < BN / 8; j++)
#pragma unroll
        for (int h = 0; h < 2; h++)
          store_pair<OutT>(pc, row0 + 8 * h, col0 + 8 * j, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], fold, it.part > 0,
                           al, be, 0, ce, 0.f, 0.f);
      if (w >= p.full_tiles && p.split > 1) {          // publish this part (the last one re-arms the flag)
        __threadfence();
        __syncwarp();
        if (lane == 0) {
          const int nv = it.part + 1 == p.split ? 0 : it.part + 1;
          asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(flag), "r"(nv) : "memory");
        }
      }
    }
  }
}

// ---- B^T for the K-major operands of tf32 / int8 ------------------------------------------------------
// src: rows x cols (pitch ld), dst: cols x rows (pitch dld).  32 x 32 tiles through shared memory; a block takes
// the row tiles blockIdx.y, + gridDim.y, ... (gridDim.y is capped at 65535: one tile unless rows > 2097120).
template <typename E>
__global__ void __launch_bounds__(256) transpose_kernel(const E* __restrict__ src, long long ld, int rows, int cols,
                                                        E* __restrict__ dst, long long dld) {
  __shared__ E tile[32][33];
  griddep_launch();
  griddep_wait();
  const int c0 = blockIdx.x * 32, rtiles = (int)(((long long)rows + 31) / 32);
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int rt = blockIdx.y; rt < rtiles; rt += gridDim.y) {
    const int r0 = rt * 32;
    if (rt != (int)blockIdx.y) __syncthreads();        // the previous tile's reads of `tile` are done
#pragma unroll
    for (int i = 0; i < 32; i += 8) {
      const int r = r0 + ty + i, c = c0 + tx;
      if (r < rows && c < cols) tile[ty + i][tx] = src[(long long)r * ld + c];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 32; i += 8) {
      const int c = c0 + ty + i, r = r0 + tx;
      if (c < cols && r < rows) dst[(long long)c * dld + r] = tile[tx][ty + i];
    }
  }
}

// ---- fp32 -> stacked bf16 planes (the split-precision pre-pass) -----------------------------------
// src: rows x cols fp32, pitch ld.  dst: NP planes stacked along rows, plane p at row p*plane_rows,
// pitch dld (elements, multiple of 8).  x = p1 + p2 + p3 with p1 = bf16(x), p2 = bf16(x - p1),
// p3 = bf16(x - p1 - p2); the subtractions are exact in fp32.  Rows [rows, plane_rows) and columns
// [cols, dld) of every plane are written as zero (K padding of B must contribute nothing).
// Range edges: a finite x never gets an infinite plane (|x| >= 0x7f7f8000 rounds to bf16 inf; its plane
// is clamped to +-0x7f7f, and the residual x - p1 stays exact), and a non-finite x gives p1 = x and
// zero lower planes.
struct SplitJob {
  const float* src; long long ld; int rows, cols;
  uint16_t* dst; long long dld; int plane_rows;
};

// One round-to-nearest-even bf16 plane of the pair (lo, hi), packed {hi, lo}; lo and hi become the residuals.
__device__ __forceinline__ uint32_t bf16_plane2(float& lo, float& hi) {
  uint32_t w;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(w) : "f"(hi), "f"(lo));
  const bool fin_lo = fabsf(lo) <= 3.40282347e38f, fin_hi = fabsf(hi) <= 3.40282347e38f;   // false for inf, NaN
  if (fin_lo && (w & 0x7FFFu) == 0x7F80u) w -= 1u;                    // +-inf -> +-0x7f7f
  if (fin_hi && (w & 0x7FFF0000u) == 0x7F800000u) w -= 0x10000u;
  lo = fin_lo ? lo - __uint_as_float(w << 16) : 0.f;
  hi = fin_hi ? hi - __uint_as_float(w & 0xFFFF0000u) : 0.f;
  return w;
}

// One launch splits both operands (blockIdx.z picks A or B).  A thread owns 8 consecutive columns
// (two 16-byte loads, one 16-byte store per plane) and walks rows blockIdx.y, +gridDim.y, ... two at
// a time so that 64 B of loads are in flight per thread; HBM-bound: 4 + 2*NP bytes per element.
template <int NP>
__global__ void __launch_bounds__(256) split_planes_kernel(const SplitJob ja, const SplitJob jb) {
  griddep_launch();
  griddep_wait();
  const SplitJob& jo = blockIdx.z == 0 ? ja : jb;
  const float* __restrict__ src = jo.src;
  uint16_t* __restrict__ dst = jo.dst;
  const long long ld = jo.ld, dld = jo.dld;
  const int rows = jo.rows, cols = jo.cols, plane_rows = jo.plane_rows;
  const int c = (int)(blockIdx.x * 256 + threadIdx.x) * 8;
  if (c >= dld) return;
  const bool vec = c + 8 <= cols && (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
  for (int r0 = blockIdx.y * 2; r0 < plane_rows; r0 += gridDim.y * 2) {
    float x[2][8];
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int r = r0 + u;
#pragma unroll
      for (int e = 0; e < 8; e++) x[u][e] = 0.f;
      if (r < rows) {
        const float* s = src + (long long)r * ld + c;
        if (vec) {
          const float4 v0 = __ldcs(reinterpret_cast<const float4*>(s));
          const float4 v1 = __ldcs(reinterpret_cast<const float4*>(s) + 1);
          x[u][0] = v0.x; x[u][1] = v0.y; x[u][2] = v0.z; x[u][3] = v0.w;
          x[u][4] = v1.x; x[u][5] = v1.y; x[u][6] = v1.z; x[u][7] = v1.w;
        } else {
#pragma unroll
          for (int e = 0; e < 8; e++)
            if (c + e < cols) x[u][e] = s[e];
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int r = r0 + u;
      if (r >= plane_rows) break;
#pragma unroll
      for (int pl = 0; pl < NP; pl++) {
        uint32_t w[4];
#pragma unroll
        for (int e = 0; e < 4; e++) w[e] = bf16_plane2(x[u][2 * e], x[u][2 * e + 1]);
        *reinterpret_cast<uint4*>(dst + ((long long)pl * plane_rows + r) * dld + c) = make_uint4(w[0], w[1], w[2], w[3]);
      }
    }
  }
}


// ---- scaled fp16 split (B200_F32_F16X2) ------------------------------------------------------------
// x' = x * 2^-e (e from the row maximum of A / the column maximum of B, so |x'| < 1), then
// x' = h1 + h2 with h1 = fp16(x'), h2 = fp16(x' - h1): 22 significant bits; h2 may be an fp16
// subnormal (absolute quantum 2^-24 relative to the row/column scale).  Three launches per GEMM:
// rows of A (maximum, scaling and split fused: each row is read from HBM once), column maxima of B,
// columns of B.  All HBM-bound: 4 bytes read + 4 bytes written per element (+ 4 read for B's maxima,
// mostly L2 hits on the second touch).
__device__ __forceinline__ void split_f16x8(const float (&x)[8], uint4& h1, uint4& h2) {
  uint32_t a[4], b[4];
#pragma unroll
  for (int e = 0; e < 4; e++) {
    const __half2 p = __floats2half2_rn(x[2 * e], x[2 * e + 1]);
    const float2 pf = __half22float2(p);
    const __half2 q = __floats2half2_rn(x[2 * e] - pf.x, x[2 * e + 1] - pf.y);
    a[e] = *reinterpret_cast<const uint32_t*>(&p);
    b[e] = *reinterpret_cast<const uint32_t*>(&q);
  }
  h1 = make_uint4(a[0], a[1], a[2], a[3]);
  h2 = make_uint4(b[0], b[1], b[2], b[3]);
}
__device__ __forceinline__ void load8(const float* __restrict__ s, int c, int cols, bool vec, float (&x)[8]) {
  if (vec && c + 8 <= cols) {
    const float4 v0 = __ldg(reinterpret_cast<const float4*>(s + c));
    const float4 v1 = __ldg(reinterpret_cast<const float4*>(s + c) + 1);
    x[0] = v0.x; x[1] = v0.y; x[2] = v0.z; x[3] = v0.w;
    x[4] = v1.x; x[5] = v1.y; x[6] = v1.z; x[7] = v1.w;
  } else {
#pragma unroll
    for (int e = 0; e < 8; e++) x[e] = c + e < cols ? __ldg(s + c + e) : 0.f;
  }
}

// A side: one warp per row.  VPL > 0: the row (cols <= 256 * VPL) stays in registers between the
// maximum and the split; VPL == 0: any length, second pass re-reads the row (L1 / L2 hits).
// dst: 2 planes stacked along rows (plane p at row p * plane_rows), pitch dld (multiple of 8); columns
// [cols, dld) and rows [rows, plane_rows) are written as zero.
template <int VPL>
__global__ void __launch_bounds__(256) split_f16_rows_kernel(const float* __restrict__ src, long long ld, int rows,
                                                             int cols, float* __restrict__ rmax,
                                                             uint16_t* __restrict__ dst, long long dld, int plane_rows) {
  griddep_launch();
  griddep_wait();
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const bool vec = (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < plane_rows; r += nwarps) {
    uint16_t* d1 = dst + (long long)r * dld;
    uint16_t* d2 = dst + ((long long)plane_rows + r) * dld;
    if (r >= rows) {
      for (int c = lane * 8; c < dld; c += 256) {
        *reinterpret_cast<uint4*>(d1 + c) = make_uint4(0, 0, 0, 0);
        *reinterpret_cast<uint4*>(d2 + c) = make_uint4(0, 0, 0, 0);
      }
      continue;
    }
    const float* s = src + (long long)r * ld;
    float mx = 0.f;
    if constexpr (VPL > 0) {
      float x[VPL][8];
#pragma unroll
      for (int j = 0; j < VPL; j++) {
        const int c = (j * 32 + lane) * 8;
#pragma unroll
        for (int e = 0; e < 8; e++) x[j][e] = 0.f;
        if (c < cols) load8(s, c, cols, vec, x[j]);
#pragma unroll
        for (int e = 0; e < 8; e++) mx = fmaxf(mx, fabsf(x[j][e]));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      if (lane == 0) rmax[r] = mx;
      const int ex = -pow2_exp(mx);
#pragma unroll
      for (int j = 0; j < VPL; j++) {
        const int c = (j * 32 + lane) * 8;
        if (c < dld) {
#pragma unroll
          for (int e = 0; e < 8; e++) x[j][e] = scale_pow2(x[j][e], ex);
          uint4 h1, h2;
          split_f16x8(x[j], h1, h2);
          *reinterpret_cast<uint4*>(d1 + c) = h1;
          *reinterpret_cast<uint4*>(d2 + c) = h2;
        }
      }
    } else {
      for (int c0 = lane * 8; c0 < cols; c0 += 1024) {       // 4 vectors in flight per lane
        float x[4][8];
#pragma unroll
        for (int u = 0; u < 4; u++) {
          const int c = c0 + u * 256;
#pragma unroll
          for (int e = 0; e < 8; e++) x[u][e] = 0.f;
          if (c < cols) load8(s, c, cols, vec, x[u]);
#pragma unroll
          for (int e = 0; e < 8; e++) mx = fmaxf(mx, fabsf(x[u][e]));
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      if (lane == 0) rmax[r] = mx;
      const int ex = -pow2_exp(mx);
      for (int c0 = lane * 8; c0 < dld; c0 += 512) {
        float x[2][8];
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const int c = c0 + u * 256;
#pragma unroll
          for (int e = 0; e < 8; e++) x[u][e] = 0.f;
          if (c < cols) load8(s, c, cols, vec, x[u]);
        }
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const int c = c0 + u * 256;
          if (c < dld) {
#pragma unroll
            for (int e = 0; e < 8; e++) x[u][e] = scale_pow2(x[u][e], ex);
            uint4 h1, h2;
            split_f16x8(x[u], h1, h2);
            *reinterpret_cast<uint4*>(d1 + c) = h1;
            *reinterpret_cast<uint4*>(d2 + c) = h2;
          }
        }
      }
    }
  }
}

// Column maxima of B into out[cols] (zero on entry; non-negative floats order like their bit patterns,
// so atomicMax on the uint view works).  A block walks 16 rows of a 1024-column strip: every row read is one
// contiguous 4 KB segment (DRAM page locality; the first version read 512-byte pieces of eight rows at a time
// and reached 3 TB/s), a thread keeps its 4 columns' maxima in registers, no cross-thread reduction.  gridDim.y is
// capped at 65535, so a block takes the row blocks blockIdx.y, + gridDim.y, ... (one unless rows > 1048560).
__global__ void __launch_bounds__(256) col_absmax_kernel(const float* __restrict__ src, long long ld, int rows,
                                                         int cols, unsigned int* __restrict__ out) {
  constexpr int ROWS = 16;      // all 16 row loads of a thread in flight at once (ncu: 32 rows in 4 batches of 8 reached 3 TB/s)
  griddep_launch();
  griddep_wait();
  const int c = blockIdx.x * 1024 + threadIdx.x * 4;
  if (c >= cols) return;
  const int rblocks = (int)(((long long)rows + ROWS - 1) / ROWS);
  const bool vec = (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0 && c + 4 <= cols;
  float4 mx = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int rb = blockIdx.y; rb < rblocks; rb += gridDim.y) {
    const int r0 = rb * ROWS, r1 = min(r0 + ROWS, rows);
    if (vec) {
#pragma unroll 16
      for (int r = r0; r < r1; r++) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(src + (long long)r * ld + c));
        mx.x = fmaxf(mx.x, fabsf(v.x)); mx.y = fmaxf(mx.y, fabsf(v.y));
        mx.z = fmaxf(mx.z, fabsf(v.z)); mx.w = fmaxf(mx.w, fabsf(v.w));
      }
    } else {
      for (int r = r0; r < r1; r++) {
        const float* s = src + (long long)r * ld + c;
        mx.x = fmaxf(mx.x, fabsf(s[0]));
        if (c + 1 < cols) mx.y = fmaxf(mx.y, fabsf(s[1]));
        if (c + 2 < cols) mx.z = fmaxf(mx.z, fabsf(s[2]));
        if (c + 3 < cols) mx.w = fmaxf(mx.w, fabsf(s[3]));
      }
    }
  }
  // Only a block that can raise the running maximum touches it: hundreds of row blocks hit the same 4 addresses and
  // same-address atomics serialise in L2 (ncu: this kernel sat at 37 % of peak DRAM throughput); after the first few
  // blocks almost every candidate is below the current value.  A stale (smaller) value read here only costs an atomic.
  const float m4[4] = {mx.x, mx.y, mx.z, mx.w};
#pragma unroll
  for (int e = 0; e < 4; e++)
    if (c + e < cols && __float_as_uint(m4[e]) > __ldcg(out + c + e)) atomicMax(out + c + e, __float_as_uint(m4[e]));
}

// B side: a thread owns 8 consecutive columns (their scale exponents live in registers) and walks rows
// blockIdx.y, +gridDim.y, ... two at a time.  Also re-zeroes `zero_buf` (the idle half of the double-
// buffered column maxima) for the next call.
__global__ void __launch_bounds__(256) split_f16_cols_kernel(const float* __restrict__ src, long long ld, int rows,
                                                             int cols, const float* __restrict__ cmax,
                                                             uint16_t* __restrict__ dst, long long dld, int plane_rows,
                                                             float* __restrict__ zero_buf, int zero_n) {
  griddep_launch();
  griddep_wait();
  const int c = (int)(blockIdx.x * 256 + threadIdx.x) * 8;
  if (blockIdx.y == 0 && zero_buf != nullptr) {
#pragma unroll
    for (int e = 0; e < 8; e++)
      if (c + e < zero_n) zero_buf[c + e] = 0.f;
  }
  if (c >= dld) return;
  const bool vec = (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
  int ex[8];
#pragma unroll
  for (int e = 0; e < 8; e++) ex[e] = c + e < cols ? -pow2_exp(__ldg(cmax + c + e)) : 0;
  for (int r0 = blockIdx.y * 2; r0 < plane_rows; r0 += gridDim.y * 2) {
    float x[2][8];
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int r = r0 + u;
#pragma unroll
      for (int e = 0; e < 8; e++) x[u][e] = 0.f;
      if (r < rows) load8(src + (long long)r * ld, c, cols, vec, x[u]);
    }
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int r = r0 + u;
      if (r >= plane_rows) break;
#pragma unroll
      for (int e = 0; e < 8; e++) x[u][e] = scale_pow2(x[u][e], ex[e]);
      uint4 h1, h2;
      split_f16x8(x[u], h1, h2);
      *reinterpret_cast<uint4*>(dst + (long long)r * dld + c) = h1;
      *reinterpret_cast<uint4*>(dst + ((long long)plane_rows + r) * dld + c) = h2;
    }
  }
}

}  // namespace b200
