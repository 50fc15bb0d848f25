// ptx.cuh — thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma shared-memory
// descriptors, register re-balancing, programmatic dependent launch.  No CUTLASS, no libraries.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace b200 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin on try_wait (HW-suspended wait, not a busy poll).  A watchdog turns a pipeline-protocol bug
// into a trap (sticky launch error the C ABI reports) instead of a hung GPU: no legitimate wait in
// these kernels approaches 4e9 SM cycles (~2 s).
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) { asm volatile("trap;"); }
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2D tiled load global -> shared, completion counted in bytes on `bar`.
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// 3D tiled load (inner, rows, batch): the strided-batched kernels read entry c2 of a stack of matrices.
__device__ __forceinline__ void tma_load_3d(uint32_t dst_smem, const CUtensorMap* m, uint32_t bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d_hint(uint32_t dst_smem, const CUtensorMap* m,
                                                 uint32_t bar, int c0, int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      ".L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "l"(policy)
      : "memory");
}

// ---------------------------------------------------------------- wgmma descriptors
// Shared-memory matrix descriptor of wgmma (64 bit):
//   [0,14) start>>4  [16,30) LBO>>4  [32,46) SBO>>4  [49,52) base offset (0: atoms 1 KB aligned)  [62,64) swizzle
// swizzle: 1 = 128B, 2 = 64B, 3 = 32B.  K-major operands: SBO = stride between 8-row groups, LBO unused.
// MN-major operands: LBO = stride between 64-element (128-byte) column blocks, SBO = stride between 8-row k groups.
// FP8 kinds name (A type, B type): torch._scaled_mm accepts these three pairs (not e5m2 x e5m2).
enum MmaKind { KIND_F16 = 0 /*bf16 operands*/, KIND_TF32 = 1, KIND_I8 = 2, KIND_FP16 = 3 /*fp16 operands*/,
               KIND_E4M3 = 4 /*e4m3 x e4m3*/, KIND_E4M3E5M2 = 5 /*e4m3 x e5m2*/, KIND_E5M2E4M3 = 6 /*e5m2 x e4m3*/ };
enum Swz { SWZ_128B = 1, SWZ_64B = 2 };

__device__ __forceinline__ uint64_t make_sdesc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t swz) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)swz << 62;
  return d;
}

// int32 accumulator -> int8, the arithmetic of chgemm's requant tail (aarch64-int8/int8kernel_m4.S:386-426):
// scvtf (int32 -> fp32, RNE), fmul by the row's scale, optional fadd of the row's bias (two roundings, not
// fused), fcvtas (to nearest, ties AWAY from zero, saturating, NaN -> 0), sqxtn x2 (saturate to int8).
__device__ __forceinline__ int32_t requant_s8(int32_t acc, float scale, float bias, bool has_bias) {
  float f = __fmul_rn(__int2float_rn(acc), scale);
  if (has_bias) f = __fadd_rn(f, bias);
  // Everything below is exact fp32 arithmetic on the FMA pipe (no F2I / FRND conversions, which run at a
  // quarter of the rate): clamp (results beyond +-200 saturate anyway), round to nearest-even with the
  // 1.5 * 2^23 constant, then move exact ties that went towards zero one step away from it.
  const float g = fminf(fmaxf(f, -200.0f), 200.0f);
  const float magic = 12582912.0f;
  float r = __fadd_rn(__fadd_rn(g, magic), -magic);
  if (fabsf(__fadd_rn(g, -r)) == 0.5f && fabsf(r) < fabsf(g)) r = __fadd_rn(r, copysignf(1.0f, g));
  r = fminf(fmaxf(r, -128.0f), 127.0f);
  const int32_t q = __float_as_int(__fadd_rn(r, magic)) - 0x4B400000;
  return f != f ? 0 : q;
}

// Epilogue activations of the 16-bit GEMMs (the B200_ACT_* codes of b200gemm.h), in fp32, shared by the tensor-core
// and the generic kernel so that both routes give the same bits for the same t.  Every step is an explicit
// round-to-nearest op, so no FMA contraction can make the two inlined copies differ.
//   RELU:      t < 0 ? +0 : t (NaN and -0 pass through, as torch.relu does)
//   GELU:      t * Phi(t) = 0.5 t erfc(-t / sqrt 2): erfc keeps relative accuracy for negative t, where 1 + erf cancels
//   GELU_TANH: 0.5 t (1 + tanh(sqrt(2 / pi) (t + 0.044715 t^3)))
// Both GELUs give +inf at +inf, -0 at -inf (the limits of the function) and NaN at NaN.
enum EpiAct { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2, ACT_GELU_TANH = 3 };
template <int ACT>
__device__ __forceinline__ float epi_act(float t) {
  if constexpr (ACT == ACT_RELU) {
    return t < 0.f ? 0.f : t;
  } else if constexpr (ACT == ACT_GELU) {
    const float g = __fmul_rn(__fmul_rn(0.5f, t), erfcf(__fmul_rn(-0.707106781186547524f, t)));
    return t == -INFINITY ? -0.f : g;
  } else if constexpr (ACT == ACT_GELU_TANH) {
    const float u = __fmul_rn(0.797884560802865356f, __fmaf_rn(__fmul_rn(0.044715f, t), __fmul_rn(t, t), t));
    const float g = __fmul_rn(__fmul_rn(0.5f, t), __fadd_rn(1.f, tanhf(u)));
    return t == -INFINITY ? -0.f : g;
  } else {
    return t;
  }
}

// Register re-balancing between warpgroups (4 aligned warps): data-movement warps give registers back,
// the epilogue warps that keep a tile's running sum in registers take them.
template <int N> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// Programmatic dependent launch: launch_dependents lets the next kernel in the stream (if it was launched with
// the programmatic-serialisation attribute) start its own prologue once every CTA of this grid has got here;
// griddep_wait blocks until the grid this one depends on has completed and its memory is visible.  Both are
// no-ops for launches without the attribute.  Every kernel launched with the attribute calls griddep_wait
// before its first global-memory access.
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

// ---- grouped GEMMs: the row blocks of each group, built on the device from its offsets ----------------------------
// Groups of one grouped call (b200_gemm_bf16_grouped): the shared-memory tables below hold kMaxGroups + 1 entries.
constexpr int kMaxGroups = 1024;

// Every thread of the block calls this (after griddep_wait where the kernel has one).  Group g covers rows
// [end[g], end[g + 1]) of the stacked A and C, with end[0] = 0 and end[g + 1] = min(max(offs[g], end[g]), total_m), so
// any offsets give ordered, in-range groups; block[g] counts the `rows`-row blocks of the groups before g
// (block[groups] = all of them).  Raw offsets are staged in end[], then warp 0 scans 32 groups per step: a running max
// (the clamp), the blocks of each group, and their prefix sum, each carried from one step to the next.
__device__ __forceinline__ void group_table(const int* __restrict__ offs, int groups, int total_m, int rows, int* end,
                                            int* block) {
  for (int i = threadIdx.x; i < groups; i += blockDim.x) end[i + 1] = offs[i];
  __syncthreads();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    int run_end = 0, run_blocks = 0;
    for (int base = 0; base < groups; base += 32) {
      const int g = base + lane;
      int e = max(g < groups ? end[g + 1] : 0, run_end);
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, e, d);
        if (lane >= d) e = max(e, o);
      }
      e = min(e, total_m);
      int prev = __shfl_up_sync(0xffffffffu, e, 1);
      if (lane == 0) prev = run_end;
      int b = (e - prev) / rows + ((e - prev) % rows != 0);           // no int overflow near total_m = 2^31 - 1
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, b, d);
        if (lane >= d) b += o;
      }
      if (g < groups) { end[g + 1] = e; block[g + 1] = run_blocks + b; }
      run_end = __shfl_sync(0xffffffffu, e, 31);
      run_blocks += __shfl_sync(0xffffffffu, b, 31);
    }
    if (lane == 0) { end[0] = 0; block[0] = 0; }
  }
  __syncthreads();
}

// The group of row block q < block[groups]: the last g with block[g] <= q, which is never an empty group.
__device__ __forceinline__ int group_of(const int* block, int groups, int q) {
  int lo = 0, hi = groups - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (block[mid] <= q) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

}  // namespace b200
