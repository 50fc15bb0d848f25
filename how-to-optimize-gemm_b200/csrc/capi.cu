// capi.cu — the C ABI of libb200gemm.so (include/b200gemm.h): argument checks, tensor-map
// construction and caching, kernel selection and launch.  Host-side counterpart of the reference's
// MY_MMult wrappers (cuda/MMult_cuda_12.cu:228-235; aarch64-int8/MMult_4x8_21.c:81-143).
//
// No cuBLAS, no CUTLASS, no CPU fallback: if no sm_90 device is usable every compute entry point
// fails with B200_ERR_NO_DEVICE.
#include "../../include/b200gemm.h"

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <vector>

#include "gemm_ffma.cuh"
#include "gemm_generic.cuh"
#include "gemm_mxf4.cuh"
#include "gemm_tc.cuh"
#include "fp8_quant.cuh"

using namespace b200;

namespace {

std::atomic<unsigned long long> g_launches{0};
int g_split_tail = 1;        // test/tuning hook (b200_gemm_debug_set_split_tail): 0 = whole tiles only

// Optional per-launch timing of the dominant GEMM kernel (bench.py's roofline.achieved): a pair of
// CUDA events is recorded on the launching stream around the kernel.  Off by default.
struct KernelTimer {
  static constexpr int CAP = 1024;
  bool on = false;
  int n = 0;
  cudaEvent_t ev[CAP][2] = {};
  void begin(cudaStream_t st) {
    if (!on || n >= CAP) return;
    if (!ev[n][0]) { cudaEventCreate(&ev[n][0]); cudaEventCreate(&ev[n][1]); }
    cudaEventRecord(ev[n][0], st);
  }
  void end(cudaStream_t st) {
    if (!on || n >= CAP) return;
    cudaEventRecord(ev[n][1], st);
    n++;
  }
} g_ktimer;
std::atomic<int> g_default_f32_mode{-1};
thread_local const char* t_last_kernel = "none";
struct Schedule { int tiles = 0, split = 0, full_tiles = 0, ctas = 0; };
thread_local Schedule t_last_schedule;     // of the last tensor-core launch (b200_gemm_debug_last_schedule)
int g_dbg_b_lbo = 0, g_dbg_b_sbo = 0;

// What one call asks of every launch it makes, built once by its entry point and passed down by reference.
struct Call {
  cudaStream_t st = nullptr;
  int acc = 0;                        // C += A*B (fp32 / int32 C): the accumulate contract
  int axpby = 0;                      // general epilogue C = alpha * A*B + beta * C
  float alpha = 1.f, beta = 0.f;
  const void* bias = nullptr;         // 16-bit bias / activation epilogue (b200_gemm_bf16_epi / _f16_epi), act -1 = none
  int act = -1;
  // SMs the tensor-core launches leave free (the row-panel plan sets it while a later K-slice of B is still being
  // broadcast: a persistent GEMM holding every SM would starve NCCL's copy kernels and serialise the exchange behind
  // the math, DESIGN §7).
  int sm_reserve = 0;
  bool epi() const { return act >= 0; }
};

// ---- per-device state ------------------------------------------------------------------------------
// Everything the library caches on a GPU lives in the context of THAT device (flags, split workspace,
// host-path staging buffers and streams, which kernels already had their dynamic shared memory limit
// raised), so one process may drive several GPUs (one host thread or one stream per GPU).  Two things are
// shared by all streams of a device, and each is ordered between streams by events:
//   - the split workspace and the F16X2 maxima: users are serialised by ws_mu on the host and by an event
//     recorded after the consuming GEMM on the device (a call on another stream waits for it);
//   - the K-split flag slots: a slot taken on another stream than its last user's waits for the event
//     recorded after that user's launch (take_flag_slot).
constexpr int kFlagSlots = 16;
struct Scratch { void* p = nullptr; size_t bytes = 0; };
struct HostPipe {
  bool ready = false;
  cudaStream_t h2d = nullptr, comp = nullptr, d2h = nullptr;
  cudaEvent_t in[8] = {}, done[8] = {};
  cudaError_t init() {
    if (ready) return cudaSuccess;
    cudaError_t e;
    if ((e = cudaStreamCreateWithFlags(&h2d, cudaStreamNonBlocking)) != cudaSuccess) return e;
    if ((e = cudaStreamCreateWithFlags(&comp, cudaStreamNonBlocking)) != cudaSuccess) return e;
    if ((e = cudaStreamCreateWithFlags(&d2h, cudaStreamNonBlocking)) != cudaSuccess) return e;
    for (int i = 0; i < 8; i++) {
      if ((e = cudaEventCreateWithFlags(&in[i], cudaEventDisableTiming)) != cudaSuccess) return e;
      if ((e = cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming)) != cudaSuccess) return e;
    }
    ready = true;
    return cudaSuccess;
  }
};
struct DevCtx {
  int ok = 0;          // 1 usable, -1 not usable, 0 unknown
  int sms = 0;
  int dev = -1;
  int* flags = nullptr;      // tail-split ordering flags (zero between launches), kFlagSlots rotating slots of 1024 ints
  std::mutex flag_mu;        // held from taking a slot until its launch is queued and flag_user[slot] updated
  unsigned flag_slot = 0;    // counts split launches only
  struct FlagUser {
    cudaStream_t st = nullptr;       // stream of the slot's last launch
    cudaEvent_t ev = nullptr;        // recorded on st right after that launch
    bool used = false;
  } flag_user[kFlagSlots];
  // split-precision workspace (planes of A and B, row / column maxima): cached, grow-only
  std::mutex ws_mu;
  Scratch ws;
  cudaEvent_t ws_event = nullptr;    // recorded after the last GEMM that read the workspace
  cudaStream_t ws_stream = nullptr;  // stream of that GEMM
  bool ws_busy = false;
  // F16X2: double-buffered column maxima (the idle half is re-zeroed by the pre-pass): of B, and of A^T when A is
  // given transposed (its column maxima are A's row maxima)
  struct MaxBuf {
    unsigned slot = 0;
    float* buf = nullptr;
    size_t cap = 0;
    int dirty[2] = {0, 0};          // entries of each half that may be non-zero
  } cmax, amax;
  cudaStream_t aux = nullptr;        // B's pre-pass chain runs here, beside A's on the caller's stream
  cudaEvent_t aux_fork = nullptr, aux_join = nullptr;
  // host-pointer entry points
  std::mutex host_mu;
  Scratch scr[4];
  HostPipe pipe;
  std::vector<const void*> attr_done;   // kernels whose MaxDynamicSharedMemorySize was raised on this device
};
constexpr int kMaxDevices = 64;
DevCtx g_ctx[kMaxDevices];
std::mutex g_mu;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;

thread_local DevCtx* t_ctx = nullptr;   // context of the device current on this thread (set by ensure_device)
thread_local int t_bound_dev = -1;      // device whose primary CUDA context this thread has made current

// Binds t_ctx to the CUDA device current on the calling thread, initialising its context on first use.
int ensure_device() {
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) { cudaGetLastError(); t_ctx = nullptr; return B200_ERR_NO_DEVICE; }
  // cudaGetDevice does not make a context current, and a host thread that has made no other runtime call has none:
  // the first driver call of a compute call (cuTensorMapEncodeTiled) would then fail with an invalid context.
  // cudaSetDevice makes the device's primary context current, once per thread and device.
  if (t_bound_dev != dev) {
    if (cudaSetDevice(dev) != cudaSuccess) { cudaGetLastError(); t_ctx = nullptr; return B200_ERR_NO_DEVICE; }
    t_bound_dev = dev;
  }
  DevCtx* c = &g_ctx[dev];
  t_ctx = c;
  if (c->ok == 1) return 0;
  std::lock_guard<std::mutex> lk(g_mu);
  if (c->ok == 1) return 0;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) { cudaGetLastError(); c->ok = -1; return B200_ERR_NO_DEVICE; }
  if (prop.major != 9) { c->ok = -1; return B200_ERR_NO_DEVICE; }
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess || !fn) {
      cudaGetLastError();
      c->ok = -1;
      return B200_ERR_NO_DEVICE;
    }
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  if (!c->flags) {
    if (cudaMalloc(&c->flags, kFlagSlots * 1024 * sizeof(int)) != cudaSuccess ||
        cudaMemset(c->flags, 0, kFlagSlots * 1024 * sizeof(int)) != cudaSuccess) {
      cudaGetLastError(); c->flags = nullptr; c->ok = -1; return B200_ERR_NO_DEVICE;
    }
  }
  if (!c->ws_event && cudaEventCreateWithFlags(&c->ws_event, cudaEventDisableTiming) != cudaSuccess) {
    cudaGetLastError(); c->ok = -1; return B200_ERR_NO_DEVICE;
  }
  for (auto& u : c->flag_user)
    if (!u.ev && cudaEventCreateWithFlags(&u.ev, cudaEventDisableTiming) != cudaSuccess) {
      cudaGetLastError(); u.ev = nullptr; c->ok = -1; return B200_ERR_NO_DEVICE;
    }
  c->dev = dev;
  c->sms = prop.multiProcessorCount;
  c->ok = 1;
  return 0;
}

// Raises a kernel's dynamic shared memory limit once per (kernel, device).
template <typename Kern>
int ensure_smem_attr(Kern kern, int bytes) {
  const void* key = reinterpret_cast<const void*>(kern);
  {
    std::lock_guard<std::mutex> lk(g_mu);
    for (const void* k : t_ctx->attr_done) if (k == key) return 0;
  }
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
  std::lock_guard<std::mutex> lk(g_mu);
  t_ctx->attr_done.push_back(key);
  return 0;
}

// ---- tensor-map cache: cuTensorMapEncodeTiled costs microseconds, the harness calls MY_MMult 20x
// back to back on the same operands (cuda/test_MMult.cpp:100-103).
struct MapKey {
  const void* ptr; int dtype; unsigned long long d0, d1, ld_bytes; unsigned b0, b1; int swz; int dev;
  unsigned long long d2, d2_bytes;     // 3-D maps (strided batch): entries and their stride; 0, 0 for a 2-D map
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && dtype == o.dtype && d0 == o.d0 && d1 == o.d1 && ld_bytes == o.ld_bytes &&
           b0 == o.b0 && b1 == o.b1 && swz == o.swz && dev == o.dev && d2 == o.d2 && d2_bytes == o.d2_bytes;
  }
};
struct MapEntry { MapKey key; CUtensorMap map; };
std::vector<MapEntry> g_maps;
size_t g_map_next = 0;
constexpr size_t kMapCache = 64;

// 2-D row-major tensor: dim0 (inner, contiguous) x dim1 rows with pitch ld_bytes.  entries > 0: a 3-D tensor of that
// many such matrices, entry_bytes apart, read one entry per box (box extent 1), so that the zero fill past the rows and
// the inner extent stays inside each entry.
int get_map(CUtensorMap* out, const void* ptr, CUtensorMapDataType dt, int elem_bytes,
            unsigned long long inner, unsigned long long rows, unsigned long long ld_bytes,
            unsigned box_inner, unsigned box_rows, int swizzle /*0 none, 1 = 128B, 2 = 128B atom 32B, 3 = 64B*/,
            unsigned long long entries = 0, unsigned long long entry_bytes = 0) {
  MapKey key{ptr, (int)dt, inner, rows, ld_bytes, box_inner, box_rows, swizzle, t_ctx->dev, entries, entry_bytes};
  std::lock_guard<std::mutex> lk(g_mu);
  for (auto& e : g_maps)
    if (e.key == key) { *out = e.map; return 0; }
  cuuint64_t dims[3] = {inner, rows, entries};
  cuuint64_t strides[2] = {ld_bytes, entry_bytes};
  cuuint32_t box[3] = {box_inner, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUtensorMap m;
  CUresult r = g_encode(&m, dt, entries ? 3 : 2, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle == 1 ? CU_TENSOR_MAP_SWIZZLE_128B
                        : swizzle == 2 ? CU_TENSOR_MAP_SWIZZLE_128B_ATOM_32B
                        : swizzle == 3 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  (void)elem_bytes;
  if (r != CUDA_SUCCESS) return B200_ERR_TENSORMAP;
  if (g_maps.size() < kMapCache) g_maps.push_back({key, m});
  else { g_maps[g_map_next] = {key, m}; g_map_next = (g_map_next + 1) % kMapCache; }
  *out = m;
  return 0;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// op_a / op_b: B200_OP_N (A is m x k, lda >= k; B is k x n, ldb >= n) or B200_OP_T (A stored as k x m, lda >= m;
// B stored as n x k, ldb >= k).
int check_args(int m, int n, int k, const void* A, int lda, const void* B, int ldb, const void* C, int ldc,
               int op_a = B200_OP_N, int op_b = B200_OP_N) {
  if ((op_a != B200_OP_N && op_a != B200_OP_T) || (op_b != B200_OP_N && op_b != B200_OP_T)) return B200_ERR_BAD_ARG;
  if (m < 0 || n < 0 || k < 0) return B200_ERR_BAD_ARG;
  if (m == 0 || n == 0) return 1;            // nothing to do
  if (!C || ldc < n) return B200_ERR_BAD_ARG;
  if (k > 0 && (!A || !B || lda < (op_a ? m : k) || ldb < (op_b ? k : n))) return B200_ERR_BAD_ARG;
  return 0;
}

int last_launch_status() {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
  return 0;
}

// Launch with the programmatic-serialisation (PDL) attribute: the kernel may start while the previous kernel of
// the stream drains; every kernel launched through here calls griddep_wait before it touches global memory.
int g_pdl = 1;                // tuning hook (b200_gemm_debug_set_pdl)
int g_prepass_fork = 1;       // F16X2: B's pre-pass chain on an auxiliary stream beside A's (b200_gemm_debug_set_pdl bit 1 = off)
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[2];
  int n = 0;
  if (cluster > 1) {
    at[n].id = cudaLaunchAttributeClusterDimension;
    at[n].val.clusterDim.x = cluster; at[n].val.clusterDim.y = 1; at[n].val.clusterDim.z = 1;
    n++;
  }
  if (g_pdl) {
    at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[n].val.programmaticStreamSerializationAllowed = 1;
    n++;
  }
  cfg.attrs = at; cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

// gridDim.y may not exceed 65535.  A y extent sized from a problem dimension (rows of C, K of a transposed operand) is
// capped here and its kernel walks y with a grid stride, so every size the ABI accepts launches; below the cap the
// grid is the uncapped one and the kernel's loop runs once.
constexpr long long kMaxGridY = 65535;
inline unsigned grid_y(long long blocks) { return (unsigned)(blocks < kMaxGridY ? blocks : kMaxGridY); }

template <typename T>
int launch_zero(int m, int n, T* C, int ldc, cudaStream_t st) {
  dim3 grid((n + 255) / 256, m < 4096 ? m : 4096);
  fill_zero_kernel<T><<<grid, 256, 0, st>>>(m, n, C, ldc);
  g_launches++;
  t_last_kernel = "fill_zero";
  return last_launch_status();
}

// op_a / op_b: B200_OP_T reads the operand as stored transposed (element strides (1, ld) instead of (ld, 1)).
template <typename InT, typename OutT>
int launch_generic(int op_a, int op_b, int m, int n, int k, const void* A, int lda, const void* B, int ldb, void* C,
                   int ldc, const char* name, const Call& c) {
  const long long mblocks = (m + 63LL) / 64;
  dim3 grid((n + 63) / 64, grid_y(mblocks));
  const long long a_rs = op_a ? 1 : lda, a_cs = op_a ? lda : 1, b_rs = op_b ? 1 : ldb, b_cs = op_b ? ldb : 1;
  auto kern = mblocks > kMaxGridY ? gemm_generic_kernel<InT, OutT, true> : gemm_generic_kernel<InT, OutT>;
  kern<<<grid, 256, 0, c.st>>>(m, n, k, static_cast<const InT*>(A), a_rs, a_cs, static_cast<const InT*>(B), b_rs, b_cs,
                               static_cast<OutT*>(C), ldc, c.acc, nullptr, nullptr, c.axpby, c.alpha, c.beta,
                               static_cast<const InT*>(c.bias), c.act);
  g_launches++;
  t_last_kernel = name;
  return last_launch_status();
}

int launch_generic_requant(int m, int n, int k, const int8_t* A, int lda, const int8_t* B, int ldb, int8_t* C,
                           int ldc, const float* scales, const float* bias, cudaStream_t st) {
  const long long mblocks = (m + 63LL) / 64;
  dim3 grid((n + 63) / 64, grid_y(mblocks));
  auto kern = mblocks > kMaxGridY ? gemm_generic_kernel<int8_t, int8_t, true> : gemm_generic_kernel<int8_t, int8_t>;
  kern<<<grid, 256, 0, st>>>(m, n, k, A, lda, 1, B, ldb, 1, C, ldc, 0, scales, bias, 0, 1.f, 0.f, nullptr, -1);
  g_launches++;
  t_last_kernel = "generic_s8_requant_64x64";
  return last_launch_status();
}

// ---- K-split flag slots --------------------------------------------------------------------
// Every launch with split > 1 takes the next of the device's kFlagSlots slots, whatever its stream, and clears it
// on its stream before the kernel runs.  Parts > 0 of a split tile spin until its flag reaches their part number.
// So a slot that comes back while its previous launch still runs on another stream must not be cleared or
// published into before that launch is done: the clear would strand a waiting part, and a publish would let it fold
// into C before the parts ahead of it had stored.  The caller holds t_ctx->flag_mu from here until
// release_flag_slot, so that two host threads never take one slot and the next taker sees this launch's event.
// On the slot's stream of last use nothing is waited for: stream order already serialises the two launches.
// Under stream capture nothing is waited for or recorded (an event recorded outside the capture cannot be waited
// on inside it), and *user stays null: a replayed graph is not ordered against split launches on other streams.
int take_flag_slot(cudaStream_t st, int** flags, DevCtx::FlagUser** user) {
  DevCtx* c = t_ctx;
  const unsigned slot = c->flag_slot++ % kFlagSlots;
  *flags = c->flags + slot * 1024;
  *user = nullptr;
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) { cudaGetLastError(); cs = cudaStreamCaptureStatusActive; }
  DevCtx::FlagUser* u = &c->flag_user[slot];
  cudaError_t e;
  if (cs == cudaStreamCaptureStatusNone) {
    // the per-thread default stream is one handle for a different stream on every host thread
    if (u->used && (u->st != st || st == cudaStreamPerThread) && (e = cudaStreamWaitEvent(st, u->ev, 0)) != cudaSuccess) {
      cudaGetLastError();
      return (int)e;
    }
    *user = u;
  }
  // the ordering flags start from zero whatever an aborted earlier launch left behind
  if ((e = cudaMemsetAsync(*flags, 0, 1024 * sizeof(int), st)) != cudaSuccess) { cudaGetLastError(); return (int)e; }
  return 0;
}
// Records the event the slot's next taker on another stream waits for: right after the launch (whether or not it
// was accepted: the clear before it was queued).
void release_flag_slot(DevCtx::FlagUser* u, cudaStream_t st) {
  if (!u) return;
  if (cudaEventRecord(u->ev, st) != cudaSuccess) { cudaGetLastError(); return; }
  u->st = st;
  u->used = true;
}

// ---- tensor-core launch -------------------------------------------------------------------
int g_force_bn = 0;          // test/tuning hook (b200_gemm_debug_set_bn): 0 = heuristic
int g_group_rows = 0;         // tuning hook: rows per raster group of the tensor-core kernels (0 = 2048)
constexpr int kStreamCDefault = 0;
int g_stream_c = -1;          // split modes: streaming stores for C (-1 = unresolved: B200GEMM_STREAM_C or the default above)
int g_ffma_fat = -1;          // strict kernel: 1 = 128x256 fat-thread variant, 0 = 128x128, -1 = by size
int g_ffma_halves = 1;        // strict kernel: split the tail round into half tiles (tuning hook)

// Operands as stored, by layout (AL / BL, gemm_tc.cuh):
//   A K-major: m x k (a_rows_total rows, pitch lda);   A MN-major: A^T, k x m (a_rows_total rows, pitch lda)
//   B MN-major: k x n (b_rows_total rows, pitch ldb);  B K-major: B^T, n x k (b_rows_total rows, pitch ldb)
// Stacked planes (split modes) lie along the rows, plane p at row p * a_plane_rows / p * b_plane_rows.  tf32 and
// int8 take K-major A and B only (launch_tc_kmajor builds them).
// EPI: the bias / activation kernel (c.bias / c.act), which never takes the K-split tail.
// STACK: the stacked kernel (gemm_tc_stacked_kernel; 16-bit kinds, single plane) over *stk, the work of every entry in
// one launch, with A and B as 3-D tensor maps.
//   STACK_BATCH: entry b of each operand at X + b * stride (elements; 0 broadcasts A or B), and the K-split tail (fp32
//   C) on the last partial round of the whole batch.
//   STACK_GROUP: groups of rows [end_g-1, end_g) of one row-major A and C (m = total_m rows; sa = sc = 0: A and C are
//   broadcast) times B_g = B + g * sb, with the ends read on the device.  The tile rows are a bound,
//   grouped_tile_rows, and there is no K split: the host does not know the tile count.
//   STACK_KGROUP: groups of K rows [end_g-1, end_g) of one A^T and one B (k = total_k; sa = sb = 0: A and B are
//   broadcast), C_g = C + g * sc, with the ends read on the device.  The tiles are a batch's, with no K split.
// (Stacking, gemm_tc.cuh, names the forms.)
// FP8 kinds (KIND_E4M3, ...): gemm_tc_fp8_kernel with the scales and bias *scl; K-major A and B, no K split.  A
// TcBlockScale (ScaleT) selects its blockwise-scaled form, whose stages carry their scales in shared memory; STACK_GROUP
// / STACK_BATCH with a TcStackScale its stacked form (the stack as above, the rowwise scales of every entry in *scl),
// and with a TcStackBlockScale its stacked blockwise form.  A TcStackScaleQ8 / TcStackBlockScaleQ8 (FP8 C) selects
// gemm_tc_fp8_q8_stacked_kernel, the same body.
struct Stack {
  int count;               // entries of a batch, or groups
  long long sa, sb, sc;    // elements between consecutive entries of A, B and C
  const int32_t* offs;     // STACK_GROUP / STACK_KGROUP: [count] cumulative ends of the groups, on the device
};
// Upper bound of the 128-row tiles of a grouped call whatever its offsets: each group adds at most one partial tile.
long long grouped_tile_rows(int total_m, int groups) { return (total_m + 127LL) / 128 + groups; }

template <int KIND, int BN, int STAGES, typename OutT, class Prod = ProdSingle, int A_ROW_BYTES = 128, int AL = LAYOUT_K,
          int BL = KindTraits<KIND>::B_LAYOUT, bool EPI = false, int STACK = STACK_NONE, class ScaleT = TcScale>
int launch_tc(int m, int n, int k, const void* A, long long lda, int a_rows_total, int a_plane_rows,
              const void* B, long long ldb, int b_rows_total, int b_plane_rows, void* C, int ldc,
              const char* name, const Call& c, int chunk_k = 0, const float* row_max = nullptr,
              const float* col_max = nullptr, const Stack* stk = nullptr, const ScaleT* scl = nullptr) {
  using Cfg = TcConfig<KIND, BN, STAGES, Prod, A_ROW_BYTES, AL, BL>;
  using T = KindTraits<KIND>;
  constexpr bool FP8 = KIND == KIND_E4M3 || KIND == KIND_E4M3E5M2 || KIND == KIND_E5M2E4M3;
  constexpr bool BLK = std::is_same<ScaleT, TcBlockScale>::value || std::is_same<ScaleT, TcStackBlockScale>::value ||
                      std::is_same<ScaleT, TcBlockScaleQ8>::value || std::is_same<ScaleT, TcStackBlockScaleQ8>::value;
  constexpr bool STACK_Q8 = std::is_same<ScaleT, TcStackScaleQ8>::value || std::is_same<ScaleT, TcStackBlockScaleQ8>::value;
  // F16X2 (fp16 planes, several products): gemm_tc_split_kernel, whose epilogue runs behind the next tile's MMAs.
  // BF16X3 / BF16X2 stay on gemm_tc_kernel (DESIGN.md §4.2).
  constexpr bool SPLIT_F16 = KIND == KIND_FP16 && Prod::N > 1;
  static_assert(!SPLIT_F16 || (std::is_same<OutT, float>::value && !EPI && STACK == STACK_NONE), "F16X2: fp32 C");
  constexpr int smem = Cfg::SMEM_BYTES + (BLK ? STAGES * kBlkScaleStageBytes : 0);
  constexpr CUtensorMapDataType dt = KIND == KIND_F16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                   : KIND == KIND_FP16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                   : KIND == KIND_TF32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                                       : CU_TENSOR_MAP_DATA_TYPE_UINT8;
  CUtensorMap tmA, tmB;
  constexpr int kswz = A_ROW_BYTES == 128 ? 1 : 3;          // K-major rows: SWIZZLE_128B or _64B
  // 3-D maps: a broadcast operand is one entry (its entry stride is then any legal value: the matrix's own extent)
  unsigned long long ea = 0, eab = 0, eb = 0, ebb = 0;
  if constexpr (STACK != STACK_NONE) {
    const unsigned long long abytes = (unsigned long long)lda * T::ELEM, bbytes = (unsigned long long)ldb * T::ELEM;
    ea = stk->sa ? stk->count : 1; eab = stk->sa ? (unsigned long long)stk->sa * T::ELEM : a_rows_total * abytes;
    eb = stk->sb ? stk->count : 1; ebb = stk->sb ? (unsigned long long)stk->sb * T::ELEM : b_rows_total * bbytes;
  }
  int rc;
  if constexpr (Cfg::A_MN)
    rc = get_map(&tmA, A, dt, T::ELEM, m, a_rows_total, (unsigned long long)lda * T::ELEM, Cfg::MN_BOX_COLS, Cfg::BK, 1, ea,
                 eab);
  else
    rc = get_map(&tmA, A, dt, T::ELEM, k, a_rows_total, (unsigned long long)lda * T::ELEM, Cfg::BK, Cfg::BM, kswz, ea, eab);
  if (rc) return rc;
  if constexpr (!Cfg::B_MN)
    rc = get_map(&tmB, B, dt, T::ELEM, k, b_rows_total, (unsigned long long)ldb * T::ELEM, Cfg::BK, Cfg::B_BOX_ROWS, kswz,
                 eb, ebb);
  else
    rc = get_map(&tmB, B, dt, T::ELEM, n, b_rows_total, (unsigned long long)ldb * T::ELEM, Cfg::B_BOX_COLS, Cfg::BK, 1,
                 eb, ebb);
  if (rc) return rc;
  TcParams p;
  p.C = C; p.ldc = ldc; p.M = m; p.N = n; p.K = k;
  // grouped: a bound, the kernel takes each group's own count from its table
  p.tiles_m = STACK == STACK_GROUP ? (int)grouped_tile_rows(m, stk->count) : (m + Cfg::TILE_M - 1) / Cfg::TILE_M;
  p.tiles_n = (n + BN - 1) / BN;
  p.group_m = (g_group_rows > 0 ? g_group_rows : 2048) / Cfg::TILE_M;     // rows of A per raster group
  if (p.group_m < 1) p.group_m = 1;
  constexpr int OB = OutBytes<OutT>::V;
  p.vec_ok = aligned16(C) && ((long long)ldc * OB) % 16 == 0;
  if constexpr (STACK != STACK_NONE) p.vec_ok = p.vec_ok && stk->sc % (16 / OB) == 0;    // every entry's C base as aligned
  p.a_plane_rows = a_plane_rows; p.b_plane_rows = b_plane_rows;
  p.chunk_kb = chunk_k > 0 ? (chunk_k + Cfg::BK - 1) / Cfg::BK : (k + Cfg::BK - 1) / Cfg::BK;
  if (p.chunk_kb < 1) p.chunk_kb = 1;
  p.dbg_b_lbo = g_dbg_b_lbo; p.dbg_b_sbo = g_dbg_b_sbo;
  p.row_max = row_max; p.col_max = col_max;
  p.accumulate = c.acc;
  p.axpby = c.axpby; p.alpha = c.alpha; p.beta = c.beta;
  p.act = c.act;
  if constexpr (EPI) p.bias = c.bias;            // shares col_max's slot: EPI kernels are never scaled
  p.stream_c = g_stream_c < 0 ? (g_stream_c = (getenv("B200GEMM_STREAM_C") ? atoi(getenv("B200GEMM_STREAM_C")) : kStreamCDefault)) : g_stream_c;
  auto kern = [] {
    if constexpr (STACK_Q8) return gemm_tc_fp8_q8_stacked_kernel<KIND, BN, STAGES, OutT, Prod, BLK, STACK>;
    else if constexpr (FP8) return gemm_tc_fp8_kernel<KIND, BN, STAGES, OutT, Prod, BLK, STACK>;
    else if constexpr (STACK != STACK_NONE) return gemm_tc_stacked_kernel<KIND, BN, STAGES, OutT, AL, BL, STACK>;
    else if constexpr (SPLIT_F16) return gemm_tc_split_kernel<KIND, BN, STAGES, Prod, A_ROW_BYTES, AL, BL>;
    else return gemm_tc_kernel<KIND, BN, STAGES, OutT, Prod, A_ROW_BYTES, AL, BL, EPI>;
  }();
  if (int arc = ensure_smem_attr(kern, smem)) return arc;
  TcStack ts{1, 0, 0, 0, nullptr};
  if constexpr (STACK != STACK_NONE) ts = TcStack{stk->count, stk->sa ? 1 : 0, stk->sb ? 1 : 0, stk->sc, stk->offs};
  [[maybe_unused]] ScaleT fp8_scale{};          // a stacked FP8 call's TcStackScale / TcStackBlockScale takes the stack here
  if constexpr (FP8) {
    fp8_scale = *scl;
    if constexpr (STACK != STACK_NONE) fp8_scale.st = ts;
  }
  // the whole batch's tiles, or the grouped call's bound on them (the entry point checked that they and their split
  // parts fit the kernel's int index)
  int tiles = p.tiles_m * p.tiles_n * (STACK == STACK_GROUP ? 1 : ts.count);
  const int units_max = t_ctx->sms - c.sm_reserve > 2 ? t_ctx->sms - c.sm_reserve : t_ctx->sms;   // one CTA per SM
  // Wave quantisation: the last, partial round of tiles (or the only round of a small problem) is
  // cut along K so that every CTA has work: rem tiles x split parts <= units.
  const int num_kb = (k + Cfg::BK - 1) / Cfg::BK;
  const int rem = tiles % units_max;
  int split = 1;
  // an activation must see the complete sum, and a grouped call's tile count is not known here: no split.  Nor for a
  // K-grouped call, whose tiles have their groups' k-blocks, or for FP8, whose scaled epilogue must see the whole sum.
  if (!EPI && !FP8 && STACK != STACK_GROUP && STACK != STACK_KGROUP && g_split_tail && OB == 4 && rem > 0) {
    split = units_max / rem;
    if (split > 4) split = 4;
    if (split > num_kb / 8) split = num_kb / 8;       // keep >= 8 k-blocks per part
    if (split < 1) split = 1;
    if (rem * Cfg::EPI_WARPS > 1024) split = 1;       // flag slot capacity
  }
  p.split = split;
  p.full_tiles = split > 1 ? tiles - rem : tiles;
  p.flags = t_ctx->flags;                   // read by split tiles only
  std::unique_lock<std::mutex> flag_lk;     // a split launch's slot: held until its event is recorded
  DevCtx::FlagUser* flag_user = nullptr;
  if (split > 1) {
    flag_lk = std::unique_lock<std::mutex>(t_ctx->flag_mu);
    if (int rc = take_flag_slot(c.st, &p.flags, &flag_user)) return rc;
  }
  const int items = p.full_tiles + (tiles - p.full_tiles) * split;
  const int units = items < units_max ? items : units_max;
  t_last_schedule = Schedule{tiles, split, p.full_tiles, units};
  g_ktimer.begin(c.st);
  {
    cudaError_t e;
    if constexpr (FP8) e = launch_pdl(kern, dim3(units), dim3(Cfg::THREADS), smem, c.st, 1, tmA, tmB, p, fp8_scale);
    else if constexpr (STACK != STACK_NONE) e = launch_pdl(kern, dim3(units), dim3(Cfg::THREADS), smem, c.st, 1, tmA, tmB, p, ts);
    else e = launch_pdl(kern, dim3(units), dim3(Cfg::THREADS), smem, c.st, 1, tmA, tmB, p);
    release_flag_slot(flag_user, c.st);
    if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
  }
  g_ktimer.end(c.st);
  g_launches++;
  t_last_kernel = name;
  return last_launch_status();
}

// Tile width: fewest "wave x tile-time" units over the persistent grid (tile time ~ BN plus a
// fixed per-tile cost); 128 x 256 has the best operand reuse, narrower tiles quantise better.  A strided batch counts
// the tiles of all its entries (one persistent grid walks them all), a grouped call its tile bound.
int pick_bn(int m, int n, bool allow256, bool allow192 = true, int batch = 1) {
  if (g_force_bn == 128 || (g_force_bn == 192 && allow192) || (g_force_bn == 256 && allow256)) return g_force_bn;
  const int cands[3] = {256, 192, 128};
  // relative per-tile efficiency assumed for the three widths: narrower tiles re-read A from shared memory
  // more often per output column
  const double eff[3] = {1.00, 0.97, 0.80};
  int best = 128;
  double best_cost = 1e300;
  const int tm = (m + 127) / 128;
  for (int i = 0; i < 3; i++) {
    if (cands[i] == 256 && !allow256) continue;
    if (cands[i] == 192 && !allow192) continue;
    const long long tiles = (long long)tm * ((n + cands[i] - 1) / cands[i]) * batch;
    const long long waves = (tiles + t_ctx->sms - 1) / t_ctx->sms;
    const double cost = (double)waves * (cands[i] / eff[i] + 8.0);
    if (cost < best_cost) { best_cost = cost; best = cands[i]; }
  }
  return best;
}

// Calls f with Width<BN> for the tile width pick_bn chooses (int8 has no 192-wide kernel).
template <int W> struct Width {
  static constexpr int BN = W, STAGES = W == 256 ? 4 : W == 192 ? 5 : 6, idx = W == 256 ? 0 : W == 192 ? 1 : 2;
};
template <bool ALLOW192 = true, class F>
int with_width(int m, int n, F&& f, int batch = 1) {
  const int bn = pick_bn(m, n, true, ALLOW192, batch);
  if (bn == 256) return f(Width<256>());
  if constexpr (ALLOW192) if (bn == 192) return f(Width<192>());
  return f(Width<128>());
}

// Calls f with the kernel layouts (AL, BL) of (op_a, op_b) and their index: 0 = NN, 1 = NT (B given as B^T), 2 = TN
// (A given as A^T), 3 = TT.  A^T is the MN-major A, B^T the K-major B.  !ALLOW_AT: row-major A only.
template <int A_L, int B_L, int I> struct Layout { static constexpr int AL = A_L, BL = B_L, idx = I; };
template <bool ALLOW_AT = true, class F>
int with_layout(int op_a, int op_b, F&& f) {
  if (!op_a) return op_b ? f(Layout<LAYOUT_K, LAYOUT_K, 1>()) : f(Layout<LAYOUT_K, LAYOUT_MN, 0>());
  if constexpr (!ALLOW_AT) return B200_ERR_BAD_ARG;
  else return op_b ? f(Layout<LAYOUT_MN, LAYOUT_K, 3>()) : f(Layout<LAYOUT_MN, LAYOUT_MN, 2>());
}

// Kernel names by [layout index][width index].
typedef const char* const KernelNames[4][3];
#define TC_NAMES(P)                                                                                 \
  {{P "_128x256", P "_128x192", P "_128x128"}, {P "_nt_128x256", P "_nt_128x192", P "_nt_128x128"}, \
   {P "_tn_128x256", P "_tn_128x192", P "_tn_128x128"}, {P "_tt_128x256", P "_tt_128x192", P "_tt_128x128"}}

// 16-bit operands: KIND_F16 (bf16, C fp32 or bf16) and KIND_FP16 (fp16, C fp32 or fp16).  E is the generic kernel's
// element type of the kind (uint16_t holds bf16 bits).  names[16-bit C][EPI]; bat_names[16-bit C]: the strided-batched
// kernels; grp_names[16-bit C]: the grouped kernels (rows NN and NT only: A is row-major); kgrp_names[16-bit C]: the
// K-grouped kernels (row TN only).
template <int KIND> struct Kind16;
template <> struct Kind16<KIND_F16> {
  using E = uint16_t;
  using Out16 = bf16_out;
  static constexpr int OUT16 = B200_OUT_BF16;
  static constexpr const char* kGeneric = "generic_bf16_64x64";
  static constexpr const char* kGenericBat = "generic_bf16_bat_64x64";
  static constexpr KernelNames names[2][2] = {{TC_NAMES("tc_bf16"), TC_NAMES("tc_bf16_epi")},
                                              {TC_NAMES("tc_bf16_obf16"), TC_NAMES("tc_bf16_obf16_epi")}};
  static constexpr KernelNames bat_names[2] = {TC_NAMES("tc_bf16_bat"), TC_NAMES("tc_bf16_obf16_bat")};
  static constexpr const char* kGenericGrp = "generic_bf16_grp_64x64";
  static constexpr KernelNames grp_names[2] = {TC_NAMES("tc_bf16_grp"), TC_NAMES("tc_bf16_obf16_grp")};
  static constexpr const char* kGenericKgrp = "generic_bf16_kgrp_64x64";
  static constexpr KernelNames kgrp_names[2] = {TC_NAMES("tc_bf16_kgrp"), TC_NAMES("tc_bf16_obf16_kgrp")};
};
template <> struct Kind16<KIND_FP16> {
  using E = __half;
  using Out16 = f16_out;
  static constexpr int OUT16 = B200_OUT_F16;
  static constexpr const char* kGeneric = "generic_f16_64x64";
  static constexpr const char* kGenericBat = "generic_f16_bat_64x64";
  static constexpr KernelNames names[2][2] = {{TC_NAMES("tc_f16"), TC_NAMES("tc_f16_epi")},
                                              {TC_NAMES("tc_f16_of16"), TC_NAMES("tc_f16_of16_epi")}};
  static constexpr KernelNames bat_names[2] = {TC_NAMES("tc_f16_bat"), TC_NAMES("tc_f16_of16_bat")};
  static constexpr const char* kGenericGrp = "generic_f16_grp_64x64";
  static constexpr KernelNames grp_names[2] = {TC_NAMES("tc_f16_grp"), TC_NAMES("tc_f16_of16_grp")};
  static constexpr const char* kGenericKgrp = "generic_f16_kgrp_64x64";
  static constexpr KernelNames kgrp_names[2] = {TC_NAMES("tc_f16_kgrp"), TC_NAMES("tc_f16_of16_kgrp")};
};

// The 16-bit GEMM on the tensor cores (OutT float, bf16_out or f16_out): every layout is read in place by one launch.
// EPI: the bias / activation kernels.  STACK: the stacked call *stk in one launch (not with EPI; see launch_tc).
template <int KIND, typename OutT, bool EPI, int STACK = STACK_NONE>
int tc16(int op_a, int op_b, int m, int n, int k, const void* A, int lda, const void* B, int ldb, void* C, int ldc,
         const Call& c, const Stack* stk = nullptr) {
  static_assert(!(EPI && STACK != STACK_NONE), "the stacked kernels have no bias / activation epilogue");
  constexpr bool c16 = !std::is_same<OutT, float>::value;
  if constexpr (STACK == STACK_KGROUP) {        // (T, N) only: both operands MN-major, K rows of total_k each
    (void)op_a; (void)op_b;
    return with_width(m, n, [&](auto W) {
      using Wd = decltype(W);
      return launch_tc<KIND, Wd::BN, Wd::STAGES, OutT, ProdSingle, 128, LAYOUT_MN, LAYOUT_MN, false, STACK>(
          m, n, k, A, lda, k, 0, B, ldb, k, 0, C, ldc, Kind16<KIND>::kgrp_names[c16][2][Wd::idx], c, 0, nullptr,
          nullptr, stk);
    }, stk->count);
  } else {
    const KernelNames& names = STACK == STACK_BATCH ? Kind16<KIND>::bat_names[c16]
                             : STACK == STACK_GROUP ? Kind16<KIND>::grp_names[c16] : Kind16<KIND>::names[c16][EPI];
    // pick_bn: a batch's tiles are those of all its entries; a grouped call's, its bound of tile rows, one row each
    const int bn_m = STACK == STACK_GROUP ? 128 : m;
    const int bn_batch = STACK == STACK_GROUP ? (int)grouped_tile_rows(m, stk->count) : stk ? stk->count : 1;
    return with_layout<STACK != STACK_GROUP>(op_a, op_b, [&](auto L) {
      using Lay = decltype(L);
      const int ar = Lay::AL == LAYOUT_MN ? k : m, br = Lay::BL == LAYOUT_MN ? k : n;    // rows of the operands as stored
      return with_width(bn_m, n, [&](auto W) {
        using Wd = decltype(W);
        return launch_tc<KIND, Wd::BN, Wd::STAGES, OutT, ProdSingle, 128, Lay::AL, Lay::BL, EPI, STACK>(
            m, n, k, A, lda, ar, 0, B, ldb, br, 0, C, ldc, names[Lay::idx][Wd::idx], c, 0, nullptr, nullptr, stk);
      }, bn_batch);
    });
  }
}

// ---- split-precision fp32 on the tensor cores ---------------------------------------------------
// Workspace for the bf16 planes: cached, grow-only (no per-call cudaMalloc in steady state).  Calls
// in split modes are serialised on this buffer by stream order; use one stream per library instance.
// K extent accumulated inside the tensor core before folding into C (0 = whole K): [0] BF16X3, [1] BF16X2
constexpr int kSplitChunkDefault[3] = {512, 512, 1024};   // BF16X3, BF16X2, F16X2
int g_split_chunk_k[3] = {kSplitChunkDefault[0], kSplitChunkDefault[1], kSplitChunkDefault[2]};
// Grows the device's split workspace to `need` bytes.  Starts at 256 MiB (every size of the reference's
// 256..4096 sweep fits: its harness averages the first, cold call into each row, and a cudaFree +
// cudaMalloc there costs tens of ms) and at least doubles.  Growth synchronises the device (other
// streams may still read the old buffer); steady-state calls never allocate.  Caller holds ws_mu.
int split_ws_reserve(size_t need) {
  DevCtx* c = t_ctx;
  if (c->ws.bytes >= need) return B200_OK;
  size_t want = c->ws.bytes ? 2 * c->ws.bytes : ((size_t)256 << 20);
  if (want < need) want = need;
  if (c->ws.p) { cudaDeviceSynchronize(); cudaFree(c->ws.p); }
  c->ws.p = nullptr; c->ws.bytes = 0; c->ws_busy = false;
  cudaError_t e = cudaMalloc(&c->ws.p, want);
  if (e != cudaSuccess && want > need) { cudaGetLastError(); want = need; e = cudaMalloc(&c->ws.p, want); }
  if (e != cudaSuccess) { cudaGetLastError(); c->ws.p = nullptr; return (int)e; }
  c->ws.bytes = want;
  return B200_OK;
}
// One call's use of the device's split workspace: holds ws_mu, grows the buffer to `bytes`, and orders the stream
// after the last user's GEMM when that ran on another stream.  At scope exit it records the event the next
// foreign-stream user will wait on.
struct WsLease {
  std::lock_guard<std::mutex> lk;
  cudaStream_t st;
  int rc;
  WsLease(size_t bytes, cudaStream_t s) : lk(t_ctx->ws_mu), st(s), rc(split_ws_reserve(bytes)) {
    DevCtx* c = t_ctx;
    if (!rc && c->ws_busy && c->ws_stream != st) cudaStreamWaitEvent(st, c->ws_event, 0);
  }
  ~WsLease() {
    if (rc) return;
    DevCtx* c = t_ctx;
    cudaEventRecord(c->ws_event, st);
    c->ws_stream = st;
    c->ws_busy = true;
  }
  uint8_t* base() const { return static_cast<uint8_t*>(t_ctx->ws.p); }
};

// src (rows x cols, pitch ld) -> dst (cols x rows, pitch dld): one launch.
template <typename E>
int launch_transpose(const E* src, long long ld, int rows, int cols, E* dst, long long dld, cudaStream_t st) {
  const cudaError_t e = launch_pdl(transpose_kernel<E>, dim3((cols + 31) / 32, grid_y((rows + 31LL) / 32)), dim3(256), 0,
                                   st, 1, src, ld, rows, cols, dst, dld);
  g_launches++;
  if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
  return last_launch_status();
}

// Pitch (elements) of a transposed copy in the workspace whose rows hold `cols` elements: a 16-byte multiple.
inline long long pitch16(int cols, int elem) { return (((long long)cols * elem + 15) & ~15LL) / elem; }
inline size_t round1024(size_t b) { return (b + 1023) & ~(size_t)1023; }
// Workspace of the tf32 / int8 routes: B^T (n x k) at offset 0 unless B is given as B^T, then A (m x k) when A is
// given as A^T.
size_t kmajor_ws_bytes(int op_a, int op_b, int m, int n, int k, int elem) {
  const size_t b = op_b ? 0 : (size_t)n * pitch16(k, elem) * elem;
  const size_t a = op_a ? (size_t)m * pitch16(k, elem) * elem : 0;
  return a ? round1024(b) + a : b;
}

// The K-major A (m x k) and B^T (n x k) that wgmma reads for tf32, int8 and FP8, staged in the workspace `ws` laid out
// as kmajor_ws_bytes(op_a, op_b) says: a row-major B and an A given as A^T are transposed there.  So is, copied at a
// 16-byte pitch in one pass, an operand given K-major that TMA cannot describe (base or pitch not a 16-byte multiple):
// the caller passes it as op_a = T / op_b = N with `copy_a` / `copy_b` set (FP8 only; tf32 and int8 take such
// operands to the generic kernel).
template <typename E>
int stage_kmajor(int op_a, int op_b, int m, int n, int k, const void*& A, long long& lda, const void*& B, long long& ldb,
                 uint8_t* ws, cudaStream_t st, bool copy_a = false, bool copy_b = false) {
  const long long kp = pitch16(k, sizeof(E));
  if (!op_b) {
    E* d = reinterpret_cast<E*>(ws);
    if (copy_b) {                                                                                  // B^T -> B^T
      const cudaError_t e = cudaMemcpy2DAsync(d, kp * sizeof(E), B, ldb * sizeof(E), (size_t)k * sizeof(E), n,
                                              cudaMemcpyDeviceToDevice, st);
      if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
    } else if (int rc = launch_transpose<E>(static_cast<const E*>(B), ldb, k, n, d, kp, st)) {    // B -> B^T
      return rc;
    }
    B = d; ldb = kp;
  }
  if (op_a) {
    E* d = reinterpret_cast<E*>(ws + (op_b ? 0 : round1024((size_t)n * kp * sizeof(E))));
    if (copy_a) {                                                                                  // A -> A
      const cudaError_t e = cudaMemcpy2DAsync(d, kp * sizeof(E), A, lda * sizeof(E), (size_t)k * sizeof(E), m,
                                              cudaMemcpyDeviceToDevice, st);
      if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
    } else if (int rc = launch_transpose<E>(static_cast<const E*>(A), lda, k, m, d, kp, st)) {    // A^T -> A
      return rc;
    }
    A = d; lda = kp;
  }
  return 0;
}

// tf32 / int8 with any layout: wgmma reads these operand types only K-major.  B given as B^T is read in place (NT
// needs no transpose and no workspace); a row-major B, and an A given as A^T, are transposed into the workspace first.
template <int KIND, int BN, int STAGES, typename OutT>
int launch_tc_kmajor(int op_a, int op_b, int m, int n, int k, const void* A, long long lda, const void* B, long long ldb,
                     void* C, int ldc, const char* name, const Call& c, const float* row_max = nullptr,
                     const float* col_max = nullptr) {
  if (!op_a && op_b) return launch_tc<KIND, BN, STAGES, OutT>(m, n, k, A, lda, m, 0, B, ldb, n, 0, C, ldc, name, c, 0, row_max, col_max);
  using E = typename std::conditional<KIND == KIND_TF32, float, uint8_t>::type;
  WsLease ws(kmajor_ws_bytes(op_a, op_b, m, n, k, sizeof(E)), c.st);
  if (ws.rc) return ws.rc;
  if (int rc = stage_kmajor<E>(op_a, op_b, m, n, k, A, lda, B, ldb, ws.base(), c.st)) return rc;
  return launch_tc<KIND, BN, STAGES, OutT>(m, n, k, A, lda, m, 0, B, ldb, n, 0, C, ldc, name, c, 0, row_max, col_max);
}

const char* const kNamesTf32[3] = {"tc_tf32_128x256", "tc_tf32_128x192", "tc_tf32_128x128"};
int tc_tf32(int op_a, int op_b, int m, int n, int k, const void* A, int lda, const void* B, int ldb, void* C, int ldc,
            const Call& c) {
  return with_width(m, n, [&](auto W) {
    using Wd = decltype(W);
    return launch_tc_kmajor<KIND_TF32, Wd::BN, Wd::STAGES, float>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc,
                                                                kNamesTf32[Wd::idx], c);
  });
}
int tc_s8(int op_a, int op_b, int m, int n, int k, const void* A, int lda, const void* B, int ldb, void* C, int ldc,
          const Call& c) {
  return with_width<false>(m, n, [&](auto W) {
    using Wd = decltype(W);
    return launch_tc_kmajor<KIND_I8, Wd::BN, Wd::STAGES, int32_t>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc,
                                                                Wd::BN == 256 ? "tc_s8_128x256" : "tc_s8_128x128", c);
  });
}
// int8 in, int8 out through the requantising epilogue (scales / bias ride in the row_max / col_max slots)
int tc_s8_requant(int m, int n, int k, const void* A, int lda, const void* B, int ldb, void* C, int ldc,
                  const float* scales, const float* bias, const Call& c) {
  return with_width<false>(m, n, [&](auto W) {
    using Wd = decltype(W);
    return launch_tc_kmajor<KIND_I8, Wd::BN, Wd::STAGES, s8_out>(
        B200_OP_N, B200_OP_N, m, n, k, A, lda, B, ldb, C, ldc,
        Wd::BN == 256 ? "tc_s8_requant_128x256" : "tc_s8_requant_128x128", c, scales, bias);
  });
}

// Plane geometry shared by the per-call pre-pass and the pre-split B handle (b200_gemm_f32_pack_b).
inline long long plane_pitch(int cols) { return ((long long)cols + 7) & ~7LL; }   // elements, 16-byte multiple
inline int b_plane_rows(int k) { return (k + 31) & ~31; }                           // zero rows pad K to the k-block

// Splits one operand (jobs == 1) or both (jobs == 2) in a single launch.
template <int NP>
int launch_split(const SplitJob& ja, const SplitJob& jb, int jobs, cudaStream_t st) {
  const long long wide = jobs == 2 && jb.dld > ja.dld ? jb.dld : ja.dld;
  const int tall = jobs == 2 && jb.plane_rows > ja.plane_rows ? jb.plane_rows : ja.plane_rows;
  const int gx = (int)((wide + 2047) / 2048);
  int gy = (t_ctx->sms * 8 + jobs * gx - 1) / (jobs * gx);        // ~8 blocks per SM over the launch
  if (gy > (tall + 1) / 2) gy = (tall + 1) / 2;
  if (gy < 1) gy = 1;
  launch_pdl(split_planes_kernel<NP>, dim3(gx, gy, jobs), dim3(256), 0, st, 1, ja, jb);
  g_launches += 1;
  return last_launch_status();
}

// Plane geometry of one operand as stored (rows x cols, split elementwise in that layout): pitch = plane_pitch(cols);
// the K index runs along the columns (row-major A, B^T: plane_rows = rows) or along the rows (row-major B, A^T:
// planes stacked with zero rows up to b_plane_rows(k), exactly as B's are for NN).
struct PlaneGeom {
  int rows, cols, plane_rows;
  long long pitch;
  size_t bytes(int np) const { return (size_t)np * plane_rows * pitch * 2; }
};
inline PlaneGeom plane_geom(bool k_along_rows, int rows, int cols) {
  return PlaneGeom{rows, cols, k_along_rows ? b_plane_rows(rows) : rows, plane_pitch(cols)};
}
inline PlaneGeom geom_a(int op_a, int m, int k) { return op_a ? plane_geom(true, k, m) : plane_geom(false, m, k); }
inline PlaneGeom geom_b(int op_b, int k, int n) { return op_b ? plane_geom(false, n, k) : plane_geom(true, k, n); }

// Workspace of a split-mode call: planes of A at 0, planes of B after them (unless B was split earlier).
size_t split_ws_bytes(int np, int op_a, int op_b, int m, int n, int k, bool prepB = false) {
  const size_t a = round1024(geom_a(op_a, m, k).bytes(np));
  return prepB ? a : a + geom_b(op_b, k, n).bytes(np);
}

KernelNames kNamesBf16x3 = TC_NAMES("tc_bf16x3"), kNamesBf16x2 = TC_NAMES("tc_bf16x2"), kNamesF16x2 = TC_NAMES("tc_f16x2");

// prepB: bf16 planes of B split earlier by b200_gemm_f32_pack_b (then only A is split here), or null.
// op_a / op_b: operands given transposed are split in their stored layout and read by the matching kernel layout.
// The running sum and the chunk accumulator of a 64 x 128 tile both live in a consumer's registers.
template <int NP>
int gemm_f32_split(int op_a, int op_b, int m, int n, int k, const float* A, int lda, const float* B, int ldb, float* C,
                   int ldc, const uint16_t* prepB, const Call& c) {
  const PlaneGeom ga = geom_a(op_a, m, k), gb = geom_b(op_b, k, n);
  WsLease ws(split_ws_bytes(NP, op_a, op_b, m, n, k, prepB != nullptr), c.st);
  if (ws.rc) return ws.rc;
  uint16_t* pA = reinterpret_cast<uint16_t*>(ws.base());
  const uint16_t* pB = prepB ? prepB : reinterpret_cast<uint16_t*>(ws.base() + round1024(ga.bytes(NP)));
  const SplitJob ja{A, lda, ga.rows, ga.cols, pA, ga.pitch, ga.plane_rows},
                 jb{B, ldb, gb.rows, gb.cols, const_cast<uint16_t*>(pB), gb.pitch, gb.plane_rows};
  if (int rc = launch_split<NP>(ja, jb, prepB ? 1 : 2, c.st)) return rc;
  using Prod = typename std::conditional<NP == 3, ProdX3, ProdX2>::type;
  return with_layout(op_a, op_b, [&](auto L) {
    using Lay = decltype(L);
    return launch_tc<KIND_F16, 128, NP == 3 ? 4 : 6, float, Prod, 64, Lay::AL, Lay::BL>(
        m, n, k, pA, ga.pitch, NP * ga.plane_rows, ga.plane_rows, pB, gb.pitch, NP * gb.plane_rows, gb.plane_rows, C, ldc,
        (NP == 3 ? kNamesBf16x3 : kNamesBf16x2)[Lay::idx][2], c, g_split_chunk_k[NP == 3 ? 0 : 1]);
  });
}

// B200_F32_F16X2: scaled fp16 split, 3 products.  Row maxima of A and column maxima of B give exact
// power-of-two scalings that bring every operand into [-1, 1] (fp16 has 5 exponent bits); the
// epilogue multiplies them back.  Launches: rows of A (max + scale + split fused), column maxima of B,
// columns of B, GEMM.
struct F16Operand {           // one operand as two stacked fp16 planes + the maxima its scaling came from
  const uint16_t* planes;     // plane p at row p * plane_rows
  long long pitch;            // elements (multiple of 8)
  int plane_rows;
  const float* maxv;          // [rows of A] / [columns of B]
};

// A (rows x cols, scaled by row) -> planes + rmax.  One launch, each row read from HBM once.
int launch_f16_split_rows(const float* A, long long lda, int rows, int cols, float* rmax, uint16_t* planes,
                          long long pitch, int plane_rows, cudaStream_t st) {
  int blocks = (plane_rows + 7) / 8;                       // one warp per row, 8 rows per block
  const int cap = t_ctx->sms * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (cols <= 1024) launch_pdl(split_f16_rows_kernel<4>, dim3(blocks), dim3(256), 0, st, 1, A, (long long)lda, rows, cols, rmax, planes, pitch, plane_rows);
  else if (cols <= 2048) launch_pdl(split_f16_rows_kernel<8>, dim3(blocks), dim3(256), 0, st, 1, A, (long long)lda, rows, cols, rmax, planes, pitch, plane_rows);
  else if (cols <= 4096) launch_pdl(split_f16_rows_kernel<16>, dim3(blocks), dim3(256), 0, st, 1, A, (long long)lda, rows, cols, rmax, planes, pitch, plane_rows);
  else launch_pdl(split_f16_rows_kernel<0>, dim3(blocks), dim3(256), 0, st, 1, A, (long long)lda, rows, cols, rmax, planes, pitch, plane_rows);
  g_launches++;
  return last_launch_status();
}

// B (rows x cols, scaled by column) -> planes + cmax (must be zero on entry).  Two launches, both made even when the
// first fails (the second clears zero_buf, which the caller counts on), and the first failure returned.  zero_buf:
// another buffer to clear on the way (the idle half of the double-buffered maxima), or null.
int launch_f16_split_cols(const float* B, long long ldb, int rows, int cols, float* cmax, uint16_t* planes,
                          long long pitch, int plane_rows, float* zero_buf, int zero_n, cudaStream_t st) {
  const cudaError_t e1 = launch_pdl(col_absmax_kernel, dim3((cols + 1023) / 1024, grid_y((rows + 15LL) / 16)), dim3(256), 0,
                                    st, 1, B, (long long)ldb, rows, cols, reinterpret_cast<unsigned int*>(cmax));
  const int gx = (int)((pitch + 2047) / 2048);
  int gy = (t_ctx->sms * 8 + gx - 1) / gx;
  if (gy > (plane_rows + 1) / 2) gy = (plane_rows + 1) / 2;
  if (gy < 1) gy = 1;
  if (zero_buf && zero_n > gx * 2048) {                    // wider than this launch covers: clear it separately
    cudaMemsetAsync(zero_buf, 0, (size_t)zero_n * 4, st);
    zero_buf = nullptr;
  }
  const cudaError_t e2 = launch_pdl(split_f16_cols_kernel, dim3(gx, gy), dim3(256), 0, st, 1, B, (long long)ldb, rows, cols, (const float*)cmax, planes, pitch, plane_rows, zero_buf, zero_n);
  g_launches += 2;
  if (e1 != cudaSuccess || e2 != cudaSuccess) { cudaGetLastError(); return (int)(e1 != cudaSuccess ? e1 : e2); }
  return last_launch_status();
}

// The F16X2 GEMM on split operands in any layout: planes of A^T are MN-major A, planes of B^T K-major B.
int gemm_f16x2_core(int op_a, int op_b, int m, int n, int k, const F16Operand& a, const F16Operand& b, float* C, int ldc,
                    const Call& c) {
  constexpr int NP = 2;
  return with_layout(op_a, op_b, [&](auto L) {
    using Lay = decltype(L);
    return launch_tc<KIND_FP16, 128, 6, float, ProdX2, 64, Lay::AL, Lay::BL>(
        m, n, k, a.planes, a.pitch, NP * a.plane_rows, a.plane_rows, b.planes, b.pitch, NP * b.plane_rows, b.plane_rows, C,
        ldc, kNamesF16x2[Lay::idx][2], c, g_split_chunk_k[2], a.maxv, b.maxv);
  });
}

// Column maxima are double-buffered outside the grow-only workspace: call i accumulates into half i % 2
// (atomicMax needs zeros) and its split launch re-zeroes the other half for call i + 1.  mb is the context's
// cmax (B's column maxima) or amax (A^T's column maxima).
int cmax_reserve(DevCtx::MaxBuf& mb, int n, float** cur, float** other, int* other_dirty) {
  if (mb.cap < (size_t)n) {
    size_t cap = mb.cap ? 2 * mb.cap : 16384;
    if (cap < (size_t)n) cap = (size_t)n;
    if (mb.buf) { cudaDeviceSynchronize(); cudaFree(mb.buf); }
    mb.buf = nullptr; mb.cap = 0;
    cudaError_t e = cudaMalloc(&mb.buf, 2 * cap * sizeof(float));
    if (e == cudaSuccess) e = cudaMemset(mb.buf, 0, 2 * cap * sizeof(float));
    if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
    mb.cap = cap;
    mb.dirty[0] = mb.dirty[1] = 0;
  }
  const unsigned slot = mb.slot++ & 1u;
  *cur = mb.buf + slot * mb.cap;
  *other = mb.buf + (slot ^ 1u) * mb.cap;
  *other_dirty = mb.dirty[slot ^ 1u];
  mb.dirty[slot ^ 1u] = 0;
  mb.dirty[slot] = n;
  return 0;
}

// Workspace of an F16X2 call: planes of A at 0, planes of B at a_off, A's row maxima at r_off (row-major A),
// B^T's row maxima at rb_off (B given as B^T).  A^T's maxima live in the double-buffered DevCtx::amax.
struct F16Ws {
  PlaneGeom ga, gb;
  size_t a_off, r_off, rb_off, total;
};
F16Ws f16x2_ws(int op_a, int op_b, int m, int n, int k, bool prepA, bool prepB) {
  F16Ws w{geom_a(op_a, m, k), geom_b(op_b, k, n)};
  w.a_off = round1024(prepA ? 0 : w.ga.bytes(2));
  w.r_off = round1024(w.a_off + (prepB ? 0 : w.gb.bytes(2)));
  const size_t ra = prepA || op_a ? 0 : (size_t)m * 4;
  w.rb_off = round1024(w.r_off + ra);
  w.total = prepB || !op_b ? w.r_off + ra : w.rb_off + (size_t)n * 4;
  return w;
}

// prepA / prepB: operands split earlier (b200_gemm_f32_pack_a / _pack_b), or null = split here.
// op_a / op_b: an operand given transposed swaps the roles of the two pre-pass kernels.  A^T (k x m) has A's row
// maxima as its column maxima: col_absmax_kernel + split_f16_cols_kernel, planes k x m (MN-major A).  B^T (n x k)
// has B's column maxima as its row maxima: split_f16_rows_kernel, planes n x k (K-major B).  The maxima are taken
// over the same sets and the split is elementwise, so the planes hold the values of the NN call's planes.
int gemm_f32_split_f16(int op_a, int op_b, int m, int n, int k, const float* A, int lda, const float* B, int ldb, float* C,
                       int ldc, const F16Operand* prepA, const F16Operand* prepB, const Call& c) {
  if (prepA && prepB) return gemm_f16x2_core(B200_OP_N, B200_OP_N, m, n, k, *prepA, *prepB, C, ldc, c);
  const F16Ws w = f16x2_ws(op_a, op_b, m, n, k, prepA != nullptr, prepB != nullptr);
  const PlaneGeom &ga = w.ga, &gb = w.gb;
  WsLease ws(w.total, c.st);
  if (ws.rc) return ws.rc;
  uint8_t* base = ws.base();
  F16Operand oa, ob;
  // Neither pre-pass kernel saturates HBM on its own (ncu: 37-52 % of peak DRAM throughput each), and A's and B's
  // chains are independent: when both operands are split here, B's chain (column maxima, split) runs on the
  // context's auxiliary stream beside A's row split and joins before the GEMM.
  DevCtx* dc = t_ctx;
  const bool fork = !prepA && !prepB && g_prepass_fork && (double)m * k + (double)k * n >= 4.0e6;
  cudaStream_t sb = c.st;
  if (fork) {
    if (!dc->aux) {
      if (cudaStreamCreateWithFlags(&dc->aux, cudaStreamNonBlocking) != cudaSuccess ||
          cudaEventCreateWithFlags(&dc->aux_fork, cudaEventDisableTiming) != cudaSuccess ||
          cudaEventCreateWithFlags(&dc->aux_join, cudaEventDisableTiming) != cudaSuccess) { cudaGetLastError(); return B200_ERR_NO_DEVICE; }
    }
    cudaEventRecord(dc->aux_fork, c.st);
    cudaStreamWaitEvent(dc->aux, dc->aux_fork, 0);
    sb = dc->aux;
  }
  if (prepB) ob = *prepB;
  else if (op_b) {
    uint16_t* pB = reinterpret_cast<uint16_t*>(base + w.a_off);
    float* bmax = reinterpret_cast<float*>(base + w.rb_off);
    if (int rc = launch_f16_split_rows(B, ldb, n, k, bmax, pB, gb.pitch, gb.plane_rows, sb)) return rc;
    ob = F16Operand{pB, gb.pitch, gb.plane_rows, bmax};
  } else {
    uint16_t* pB = reinterpret_cast<uint16_t*>(base + w.a_off);
    float *cmax, *other;
    int other_dirty;
    if (int rc = cmax_reserve(dc->cmax, n, &cmax, &other, &other_dirty)) return rc;
    if (int rc = launch_f16_split_cols(B, ldb, k, n, cmax, pB, gb.pitch, gb.plane_rows, other, other_dirty, sb)) return rc;
    ob = F16Operand{pB, gb.pitch, gb.plane_rows, cmax};
  }
  if (prepA) oa = *prepA;
  else if (op_a) {
    uint16_t* pA = reinterpret_cast<uint16_t*>(base);
    float *amax, *other;
    int other_dirty;
    if (int rc = cmax_reserve(dc->amax, m, &amax, &other, &other_dirty)) return rc;
    if (int rc = launch_f16_split_cols(A, lda, k, m, amax, pA, ga.pitch, ga.plane_rows, other, other_dirty, c.st)) return rc;
    oa = F16Operand{pA, ga.pitch, ga.plane_rows, amax};
  } else {
    uint16_t* pA = reinterpret_cast<uint16_t*>(base);
    float* rmax = reinterpret_cast<float*>(base + w.r_off);
    if (int rc = launch_f16_split_rows(A, lda, m, k, rmax, pA, ga.pitch, ga.plane_rows, c.st)) return rc;
    oa = F16Operand{pA, ga.pitch, ga.plane_rows, rmax};
  }
  if (fork) {
    cudaEventRecord(dc->aux_join, dc->aux);
    cudaStreamWaitEvent(c.st, dc->aux_join, 0);
  }
  return gemm_f16x2_core(op_a, op_b, m, n, k, oa, ob, C, ldc, c);
}

// The strict FFMA kernels (gemm_ffma.cuh) on TMA-able row-major operands, ctas_per_sm CTAs of Cfg per SM: tiles of
// the last, at most half-full round are issued as two half tiles each.
template <class Cfg, class Kern>
int launch_ffma(Kern kern, int ctas_per_sm, const char* name, int m, int n, int k, const float* A, int lda,
                const float* B, int ldb, float* C, int ldc, const Call& c) {
  CUtensorMap tmA, tmB;
  int rc = get_map(&tmA, A, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, k, m, (unsigned long long)lda * 4, Cfg::BK, Cfg::BM, 1);
  if (rc) return rc;
  rc = get_map(&tmB, B, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, n, k, (unsigned long long)ldb * 4, Cfg::BN, Cfg::BK, 0);
  if (rc) return rc;
  FfmaParams p;
  p.C = C; p.ldc = ldc; p.M = m; p.N = n; p.K = k;
  p.vec_ok = aligned16(C) && (ldc % 4) == 0;
  p.accumulate = c.acc;
  p.axpby = c.axpby; p.alpha = c.alpha; p.beta = c.beta;
  p.tiles_m = (m + Cfg::BM - 1) / Cfg::BM;
  p.tiles_n = (n + Cfg::BN - 1) / Cfg::BN;
  p.group_m = 8;
  const int tiles = p.tiles_m * p.tiles_n, slots = ctas_per_sm * t_ctx->sms;
  const int rem = tiles % slots;
  const bool halves = g_ffma_halves && rem > 0 && 2 * rem <= slots;
  p.full_tiles = halves ? tiles - rem : tiles;
  const int ctas = p.full_tiles + 2 * (tiles - p.full_tiles);
  if (int arc = ensure_smem_attr(kern, Cfg::SMEM_BYTES)) return arc;
  g_ktimer.begin(c.st);
  kern<<<ctas, Cfg::THREADS, Cfg::SMEM_BYTES, c.st>>>(tmA, tmB, p);
  g_ktimer.end(c.st);
  g_launches++;
  t_last_kernel = name;
  return last_launch_status();
}

// STRICT with a transposed operand: the FFMA kernels read row-major A and B, so A^T / B^T are first transposed into
// the workspace (A at 0, then B; 16-byte pitches).  The kernel and its arithmetic are those of NN.
size_t strict_ws_bytes(int op_a, int op_b, int m, int n, int k) {
  const size_t a = op_a ? (size_t)m * pitch16(k, 4) * 4 : 0, b = op_b ? (size_t)k * pitch16(n, 4) * 4 : 0;
  return a && b ? round1024(a) + b : a + b;
}
// The strict kernel for TMA-able operands: 128x256 fat-thread tiles from 96 of them (measured on H100, fat : 128x128
// TFLOP/s — 4096^3 45.6 : 43.8, 3072^3 40.4 : 43.1, 2048^3 43.5 : 42.8, 1536^3 25.2 : 24.0; at 1024^3, 32 fat tiles,
// the small tile wins 36.2 : 20.1)
int strict_tma(int op_a, int op_b, int m, int n, int k, const float* A, int lda, const float* B, int ldb, float* C,
               int ldc, const Call& c) {
  if (op_a || op_b) {
    WsLease ws(strict_ws_bytes(op_a, op_b, m, n, k), c.st);
    if (ws.rc) return ws.rc;
    const long long kp = pitch16(k, 4), np = pitch16(n, 4);
    if (op_a) {
      float* a = reinterpret_cast<float*>(ws.base());
      if (int rc = launch_transpose<float>(A, lda, k, m, a, kp, c.st)) return rc;          // A^T (k x m) -> A (m x k)
      A = a; lda = (int)kp;
    }
    if (op_b) {
      float* b = reinterpret_cast<float*>(ws.base() + (op_a ? round1024((size_t)m * kp * 4) : 0));
      if (int rc = launch_transpose<float>(B, ldb, n, k, b, np, c.st)) return rc;          // B^T (n x k) -> B (k x n)
      B = b; ldb = (int)np;
    }
    return strict_tma(B200_OP_N, B200_OP_N, m, n, k, A, lda, B, ldb, C, ldc, c);
  }
  if (g_ffma_fat == 1 || (g_ffma_fat < 0 && (long long)((m + 127) / 128) * ((n + 255) / 256) >= 96))
    return launch_ffma<FfmaFatCfg>(gemm_ffma_fat_kernel, 1, "ffma_fat_128x256x32_tma", m, n, k, A, lda, B, ldb, C, ldc, c);
  return launch_ffma<FfmaCfg>(gemm_ffma_kernel, 2, "ffma_128x128x32_tma", m, n, k, A, lda, B, ldb, C, ldc, c);
}

bool tma_ok(const void* A, int lda, const void* B, int ldb, int elem) {
  return aligned16(A) && aligned16(B) && ((long long)lda * elem) % 16 == 0 && ((long long)ldb * elem) % 16 == 0;
}

int resolve_f32_mode(int mode) {
  if (mode == B200_F32_AUTO) {
    int d = g_default_f32_mode.load();
    if (d < 0) {
      const char* e = getenv("B200GEMM_F32_MODE");
      d = e ? atoi(e) : B200_F32_F16X2;
      if (d < 0 || d == B200_F32_AUTO || d > B200_F32_F16X2) d = B200_F32_F16X2;
      g_default_f32_mode.store(d);
    }
    return d;
  }
  return mode;
}

enum F32Route { R_NONE, R_GENERIC, R_STRICT, R_TF32, R_BF16X3, R_BF16X2, R_F16X2 };

// The route of an fp32 call: `mode` as requested, tma = tma_ok of the operands as stored, general = a general
// (alpha, beta).  AUTO takes the default mode d, except where the first matching row below says otherwise:
//   tma, m*n*k <= 2e8, and general or d in {BF16X3, F16X2}   -> STRICT
//   not general, d == F16X2, m*n*k < 1.3e9                   -> BF16X3
// STRICT and TF32 on operands that are not TMA-able take the generic CUDA-core kernel; an unknown mode has no route.
// AUTO on a small problem: the split path costs two launches (pre-pass + GEMM); up to 512^3 the single-launch strict
// FFMA kernel keeps up with it and is bit-exact against the reference oracle (measured on H100 with
// tools/probe_crossover.py, TFLOP/s strict : BF16X3 — 256^3 1.9 : 2.0, 512^3 8.6 : 8.4); from 640^3 the tensor-core
// path pulls away (13.6 : 14.9, 1024^3 36.4 : 51.4).
// AUTO between ~640^3 and ~1100^3: the two-launch BF16X3 path (one fused split + GEMM) beats the four-launch F16X2
// path while launches, not tensor work, dominate (H100, TFLOP/s BF16X3 : F16X2 — 768^3 20.3 : 15.3, 1024^3
// 51.4 : 42.6, 1152^3 65.8 : 72.3, 2048^3 109 : 146).  Both are fp32-class.
F32Route f32_route(int mode, int m, int n, int k, bool tma, bool general) {
  const double mnk = (double)m * n * k;
  int d = resolve_f32_mode(mode);
  if (mode == B200_F32_AUTO) {
    if (tma && mnk <= 2.0e8 && (general || d == B200_F32_BF16X3 || d == B200_F32_F16X2)) d = B200_F32_STRICT;
    else if (!general && d == B200_F32_F16X2 && mnk < 1.3e9) d = B200_F32_BF16X3;
  }
  switch (d) {
    case B200_F32_STRICT: return tma ? R_STRICT : R_GENERIC;
    case B200_F32_TF32: return tma ? R_TF32 : R_GENERIC;
    case B200_F32_BF16X3: return R_BF16X3;
    case B200_F32_BF16X2: return R_BF16X2;
    case B200_F32_F16X2: return R_F16X2;
    default: return R_NONE;
  }
}

// Workspace the route reserves for one call.
size_t f32_route_ws_bytes(F32Route r, int op_a, int op_b, int m, int n, int k) {
  switch (r) {
    case R_STRICT: return strict_ws_bytes(op_a, op_b, m, n, k);
    case R_TF32: return kmajor_ws_bytes(op_a, op_b, m, n, k, 4);
    case R_BF16X3: return split_ws_bytes(3, op_a, op_b, m, n, k);
    case R_BF16X2: return split_ws_bytes(2, op_a, op_b, m, n, k);
    case R_F16X2: return f16x2_ws(op_a, op_b, m, n, k, false, false).total;
    default: return 0;
  }
}

// k == 0 or alpha == 0: C = act(beta * C + bias) without reading A or B, in one pass (none for the accumulate
// contract); beta == 0 does not read C.  T: the element type of C; BE: the bias type of a 16-bit call, void for the
// others (fp32 C has no bias / activation epilogue).
template <typename T, typename BE>
int degenerate(int m, int n, void* C, int ldc, const Call& c) {
  const dim3 grid((n + 255) / 256, m < 4096 ? m : 4096);
  if constexpr (!std::is_void<BE>::value) {
    if (c.epi()) {
      bias_act_inplace_kernel<T, BE><<<grid, 256, 0, c.st>>>(m, n, static_cast<T*>(C), ldc, c.beta,
                                                              static_cast<const BE*>(c.bias), c.act);
      g_launches++;
      t_last_kernel = "bias_act_inplace";
      return last_launch_status();
    }
  }
  if (c.acc) return 0;
  if (c.beta == 0.f) {          // 16-bit C is cleared as raw bits
    using Z = typename std::conditional<sizeof(T) == 2, uint16_t, T>::type;
    return launch_zero<Z>(m, n, static_cast<Z*>(C), ldc, c.st);
  }
  scale_inplace_kernel<T><<<grid, 256, 0, c.st>>>(m, n, static_cast<T*>(C), ldc, c.beta);
  g_launches++;
  return last_launch_status();
}

// fp32: C = alpha * op(A) op(B) + beta * C (the contract of the reference's cuBLAS comparator,
// cuda/MMult_cuBLAS_1.cpp:11-19).  (1, 0) is the plain call and (1, 1) the accumulate contract C += AB; any other
// pair is applied by every kernel's epilogue (alpha * AB, then + beta * C with C read only when beta != 0): no
// pre-scaled C, so beta / alpha never has to be representable.  sm_reserve: SMs the tensor-core launches leave free.
int gemm_f32(int op_a, int op_b, int m, int n, int k, float alpha, const float* A, int lda, const float* B, int ldb,
             float beta, float* C, int ldc, int mode, cudaStream_t st, int sm_reserve = 0) {
  int rc = check_args(m, n, k, A, lda, B, ldb, C, ldc, op_a, op_b);
  if (rc == 1) return 0;
  if (rc) return rc;
  if ((rc = ensure_device())) return rc;
  Call c{st};
  c.sm_reserve = sm_reserve;
  if (alpha == 1.f && (beta == 0.f || beta == 1.f)) c.acc = beta == 1.f;
  else { c.axpby = 1; c.alpha = alpha; c.beta = beta; }
  if (k == 0 || alpha == 0.f) return degenerate<float, void>(m, n, C, ldc, c);
  switch (f32_route(mode, m, n, k, tma_ok(A, lda, B, ldb, 4), c.axpby)) {
    case R_GENERIC: return launch_generic<float, float>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, "generic_f32_64x64", c);
    case R_STRICT: return strict_tma(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, c);
    case R_TF32: return tc_tf32(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, c);
    case R_BF16X3: return gemm_f32_split<3>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, nullptr, c);
    case R_BF16X2: return gemm_f32_split<2>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, nullptr, c);
    case R_F16X2: return gemm_f32_split_f16(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, nullptr, nullptr, c);
    default: return B200_ERR_UNSUPPORTED;
  }
}

// 16-bit operands: C = round_out(act(fma(beta, float(C), alpha * op(A) op(B)) + bias)).  (1, 0) without a bias or an
// activation is the plain call; a null bias with B200_ACT_NONE is the general (alpha, beta) call.  Every layout is
// read in place by one launch.
template <int KIND>
int gemm16(int op_a, int op_b, int m, int n, int k, float alpha, const uint16_t* A, int lda, const uint16_t* B, int ldb,
           float beta, void* C, int ldc, int out_type, const uint16_t* bias, int act, cudaStream_t st) {
  using K16 = Kind16<KIND>;
  using E = typename K16::E;
  if (act < B200_ACT_NONE || act > B200_ACT_GELU_TANH) return B200_ERR_BAD_ARG;
  if (out_type != B200_OUT_F32 && out_type != K16::OUT16) return B200_ERR_BAD_ARG;
  int rc = check_args(m, n, k, A, lda, B, ldb, C, ldc, op_a, op_b);
  if (rc == 1) return 0;
  if (rc) return rc;
  if ((rc = ensure_device())) return rc;
  Call c{st};
  if (bias || act != B200_ACT_NONE) { c.bias = bias; c.act = act; }
  if (c.epi() || alpha != 1.f || beta != 0.f) { c.axpby = 1; c.alpha = alpha; c.beta = beta; }
  const bool c32 = out_type == B200_OUT_F32;
  if (k == 0 || alpha == 0.f) return c32 ? degenerate<float, E>(m, n, C, ldc, c) : degenerate<E, E>(m, n, C, ldc, c);
  if (!tma_ok(A, lda, B, ldb, 2)) {
    if (c32) return launch_generic<E, float>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, K16::kGeneric, c);
    return launch_generic<E, E>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, K16::kGeneric, c);
  }
  using O16 = typename K16::Out16;
  if (c.epi()) return c32 ? tc16<KIND, float, true>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, c)
                          : tc16<KIND, O16, true>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, c);
  return c32 ? tc16<KIND, float, false>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, c)
             : tc16<KIND, O16, false>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, c);
}

// ---- strided-batched 16-bit GEMM ----------------------------------------------------------------------------------
// Grid z of the batched generic and element-wise kernels: the entries run over blockIdx.z, this many at a time.
constexpr int kMaxGridZ = 65535;

// k == 0 or alpha == 0 over every entry of a batch, one launch: C = beta * C (C unread when beta == 0).
template <typename T>
int degenerate_batched(int m, int n, void* C, int ldc, const Stack& bt, const Call& c) {
  const int gz = bt.count < kMaxGridZ ? bt.count : kMaxGridZ;
  int gy = 4096 / gz;
  if (gy > m) gy = m;
  if (gy < 1) gy = 1;
  const dim3 grid((n + 255) / 256, gy, gz);
  if (c.beta == 0.f) {          // 16-bit C is cleared as raw bits
    using Z = typename std::conditional<sizeof(T) == 2, uint16_t, T>::type;
    fill_zero_batched_kernel<Z><<<grid, 256, 0, c.st>>>(bt.count, m, n, static_cast<Z*>(C), ldc, bt.sc);
    t_last_kernel = "fill_zero_bat";
  } else {
    scale_inplace_batched_kernel<T><<<grid, 256, 0, c.st>>>(bt.count, m, n, static_cast<T*>(C), ldc, bt.sc, c.beta);
    t_last_kernel = "scale_inplace_bat";
  }
  g_launches++;
  return last_launch_status();
}

// Operands TMA cannot describe, and overlapping input entries: the CUDA-core kernel, each entry as launch_generic
// computes one matrix.
template <typename InT, typename OutT>
int launch_generic_batched(int op_a, int op_b, int m, int n, int k, const void* A, int lda, const void* B, int ldb,
                           void* C, int ldc, const Stack& bt, const char* name, const Call& c) {
  dim3 grid((n + 63) / 64, grid_y((m + 63LL) / 64), bt.count < kMaxGridZ ? bt.count : kMaxGridZ);
  const long long a_rs = op_a ? 1 : lda, a_cs = op_a ? lda : 1, b_rs = op_b ? 1 : ldb, b_cs = op_b ? ldb : 1;
  gemm_generic_batched_kernel<InT, OutT><<<grid, 256, 0, c.st>>>(
      bt.count, m, n, k, static_cast<const InT*>(A), a_rs, a_cs, bt.sa, static_cast<const InT*>(B), b_rs, b_cs, bt.sb,
      static_cast<OutT*>(C), ldc, bt.sc, c.axpby, c.alpha, c.beta);
  g_launches++;
  t_last_kernel = name;
  return last_launch_status();
}

// One operand of a batch as a 3-D tensor map: its entry stride (elements) a 16-byte multiple that TMA can encode, and
// either 0 (broadcast) or at least the entry's rows x ld, since the encoder documents each stride as covering the
// dimension before it.  Overlapping entries (0 < stride < rows x ld, which cuBLAS allows for inputs) go to the
// generic kernel.
bool batch_tma_ok(long long stride, long long rows, long long ld, int elem) {
  return stride == 0 || (stride < (1LL << 40) / elem && (stride * elem) % 16 == 0 && stride >= rows * ld);
}

// C_b = round_out(fma(beta, float(C_b), alpha * op(A_b) op(B_b))) for b < batch, X_b = X + b * stride_x (elements).
// Argument rules (all before the device is touched): those of gemm16 per entry; batch < 0 or a negative stride is
// B200_ERR_BAD_ARG; batch == 0, m == 0 or n == 0 is a no-op; batch > 1 with entries of C that overlap is
// B200_ERR_BAD_ARG, as is a batch whose tiles the kernel's int work index cannot count.  batch == 1 is the _ex call.
template <int KIND>
int gemm16_batched(int op_a, int op_b, int m, int n, int k, float alpha, const uint16_t* A, int lda, long long stride_a,
                   const uint16_t* B, int ldb, long long stride_b, float beta, void* C, int ldc, long long stride_c,
                   int batch, int out_type, cudaStream_t st) {
  using K16 = Kind16<KIND>;
  using E = typename K16::E;
  if (batch < 0 || stride_a < 0 || stride_b < 0 || stride_c < 0) return B200_ERR_BAD_ARG;
  if (out_type != B200_OUT_F32 && out_type != K16::OUT16) return B200_ERR_BAD_ARG;
  if ((op_a != B200_OP_N && op_a != B200_OP_T) || (op_b != B200_OP_N && op_b != B200_OP_T)) return B200_ERR_BAD_ARG;
  if (m < 0 || n < 0 || k < 0) return B200_ERR_BAD_ARG;
  if (batch == 0) return 0;
  if (batch == 1)
    return gemm16<KIND>(op_a, op_b, m, n, k, alpha, A, lda, B, ldb, beta, C, ldc, out_type, nullptr, B200_ACT_NONE, st);
  int rc = check_args(m, n, k, A, lda, B, ldb, C, ldc, op_a, op_b);
  if (rc == 1) return 0;
  if (rc) return rc;
  if (stride_c < (long long)(m - 1) * ldc + n) return B200_ERR_BAD_ARG;                 // entries of C would overlap
  // Offsets: the last entry of each operand within 2^60 elements, so no byte offset wraps.  Tiles: the batch's tiles
  // at the narrowest width, times up to 4 K-split parts, must fit the kernel's int work index.  Both by division.
  const long long max_stride = (1LL << 60) / (batch - 1);
  if (stride_a > max_stride || stride_b > max_stride || stride_c > max_stride) return B200_ERR_BAD_ARG;
  const long long tiles1 = ((m + 127LL) / 128) * ((n + 127LL) / 128);                  // < 2^48
  if (tiles1 > 0x7FFFFFFFLL / 4 / batch) return B200_ERR_BAD_ARG;
  if ((rc = ensure_device())) return rc;
  Call c{st};
  if (alpha != 1.f || beta != 0.f) { c.axpby = 1; c.alpha = alpha; c.beta = beta; }
  const bool c32 = out_type == B200_OUT_F32;
  const Stack bt{batch, stride_a, stride_b, stride_c, nullptr};
  if (k == 0 || alpha == 0.f) return c32 ? degenerate_batched<float>(m, n, C, ldc, bt, c) : degenerate_batched<E>(m, n, C, ldc, bt, c);
  const int ar = op_a ? k : m, br = op_b ? n : k;                                       // rows of the operands as stored
  if (!tma_ok(A, lda, B, ldb, 2) || !batch_tma_ok(stride_a, ar, lda, 2) || !batch_tma_ok(stride_b, br, ldb, 2)) {
    if (c32) return launch_generic_batched<E, float>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, bt, K16::kGenericBat, c);
    return launch_generic_batched<E, E>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, bt, K16::kGenericBat, c);
  }
  if (c32) return tc16<KIND, float, false, STACK_BATCH>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, c, &bt);
  return tc16<KIND, typename K16::Out16, false, STACK_BATCH>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, c, &bt);
}

// ---- grouped 16-bit GEMM (torch._grouped_mm) -----------------------------------------------------------------------
// The offsets stay on the device: every launch below reads them there, and the host never waits for them.  A grouped
// call is a Stack with offs set (launch_tc); total_m is its m.

// k == 0 or alpha == 0: C = beta * C (C unread when beta == 0) on rows [0, end of the last group), one launch.
template <typename T>
int degenerate_grouped(int total_m, int n, void* C, int ldc, const Stack& gr, const Call& c) {
  const dim3 grid((n + 255) / 256, total_m < 4096 ? total_m : 4096);
  if (c.beta == 0.f) {          // 16-bit C is cleared as raw bits
    using Z = typename std::conditional<sizeof(T) == 2, uint16_t, T>::type;
    fill_zero_grouped_kernel<Z><<<grid, 256, 0, c.st>>>(gr.offs, gr.count, total_m, n, static_cast<Z*>(C), ldc);
    t_last_kernel = "fill_zero_grp";
  } else {
    scale_inplace_grouped_kernel<T><<<grid, 256, 0, c.st>>>(gr.offs, gr.count, total_m, n, static_cast<T*>(C), ldc,
                                                            c.beta);
    t_last_kernel = "scale_inplace_grp";
  }
  g_launches++;
  return last_launch_status();
}

// Operands TMA cannot describe: the CUDA-core kernel, each group as launch_generic computes its rows.  The grid counts
// the 64-row blocks of every group at their upper bound; the column blocks run gridDim.y at a time.
template <typename InT, typename OutT>
int launch_generic_grouped(int op_b, int total_m, int n, int k, const void* A, int lda, const void* B, int ldb, void* C,
                           int ldc, const Stack& gr, const char* name, const Call& c) {
  const int tn = (n + 63) / 64;
  dim3 grid((int)((total_m + 63LL) / 64 + gr.count), tn < 65535 ? tn : 65535);
  const long long b_rs = op_b ? 1 : ldb, b_cs = op_b ? ldb : 1;
  gemm_generic_grouped_kernel<InT, OutT><<<grid, 256, 0, c.st>>>(
      gr.offs, gr.count, total_m, n, k, static_cast<const InT*>(A), lda, static_cast<const InT*>(B), b_rs, b_cs,
      gr.sb, static_cast<OutT*>(C), ldc, c.axpby, c.alpha, c.beta);
  g_launches++;
  t_last_kernel = name;
  return last_launch_status();
}

// Rows [end_{g-1}, end_g) of C = round_out(fma(beta, float(C), alpha * A_rows op(B_g))), B_g = B + g * stride_b, with
// end_{-1} = 0 and end_g = min(max(offs[g], end_{g-1}), total_m) on the device.  Argument rules (all before the device
// is touched, all by division): those of gemm16 for an m = total_m call with op_a = N; negative sizes or stride;
// groups > kMaxGroups; groups > 1 with B_g overlapping (stride_b < rows x ldb); (groups - 1) * stride_b above 2^60;
// a tile bound the kernel's int work index cannot count; a null offs with work to do.  groups == 0, total_m == 0 or
// n == 0 is a no-op.
template <int KIND>
int gemm16_grouped(int op_b, int total_m, int n, int k, float alpha, const uint16_t* A, int lda, const uint16_t* B,
                   int ldb, long long stride_b, const int32_t* offs, int groups, float beta, void* C, int ldc,
                   int out_type, cudaStream_t st) {
  using K16 = Kind16<KIND>;
  using E = typename K16::E;
  if (groups < 0 || stride_b < 0 || groups > kMaxGroups) return B200_ERR_BAD_ARG;
  if (out_type != B200_OUT_F32 && out_type != K16::OUT16) return B200_ERR_BAD_ARG;
  if (op_b != B200_OP_N && op_b != B200_OP_T) return B200_ERR_BAD_ARG;
  if (total_m < 0 || n < 0 || k < 0) return B200_ERR_BAD_ARG;
  if (groups == 0) return 0;
  int rc = check_args(total_m, n, k, A, lda, B, ldb, C, ldc, B200_OP_N, op_b);
  if (rc == 1) return 0;
  if (rc) return rc;
  if (!offs) return B200_ERR_BAD_ARG;
  const long long b_rows = op_b ? n : k;                                               // rows of one B_g as stored
  if (groups > 1) {
    if (stride_b < b_rows * ldb) return B200_ERR_BAD_ARG;                            // B_g would overlap
    if (stride_b > (1LL << 60) / (groups - 1)) return B200_ERR_BAD_ARG;
  }
  // the tile bound at the narrowest width, with room for w + gridDim.x, in the kernel's int work index
  const long long tiles_n = (n + 127LL) / 128;
  if (tiles_n > 0x3FFFFFFFLL / grouped_tile_rows(total_m, groups)) return B200_ERR_BAD_ARG;
  if ((rc = ensure_device())) return rc;
  Call c{st};
  if (alpha != 1.f || beta != 0.f) { c.axpby = 1; c.alpha = alpha; c.beta = beta; }
  const bool c32 = out_type == B200_OUT_F32;
  const Stack gr{groups, 0, groups > 1 ? stride_b : 0, 0, offs};
  if (k == 0 || alpha == 0.f)
    return c32 ? degenerate_grouped<float>(total_m, n, C, ldc, gr, c) : degenerate_grouped<E>(total_m, n, C, ldc, gr, c);
  if (!tma_ok(A, lda, B, ldb, 2) || (groups > 1 && !batch_tma_ok(stride_b, b_rows, ldb, 2))) {
    if (c32) return launch_generic_grouped<E, float>(op_b, total_m, n, k, A, lda, B, ldb, C, ldc, gr, K16::kGenericGrp, c);
    return launch_generic_grouped<E, E>(op_b, total_m, n, k, A, lda, B, ldb, C, ldc, gr, K16::kGenericGrp, c);
  }
  if (c32) return tc16<KIND, float, false, STACK_GROUP>(B200_OP_N, op_b, total_m, n, k, A, lda, B, ldb, C, ldc, c, &gr);
  return tc16<KIND, typename K16::Out16, false, STACK_GROUP>(B200_OP_N, op_b, total_m, n, k, A, lda, B, ldb, C, ldc, c,
                                                              &gr);
}

// ---- K-grouped 16-bit GEMM (torch._grouped_mm 2-D x 2-D: the weight gradient of a grouped layer) -------------------
// total_k: the largest K extent; every K row coordinate the kernels form, end + 64 included, stays below 2^31.
constexpr int kMaxTotalK = 0x7FFFFFFF - 64;

// Layouts other than (T, N) and operands TMA cannot describe: the CUDA-core kernel, each group as launch_generic
// computes C_g from copies of its K range.
template <typename InT, typename OutT>
int launch_generic_kgrouped(int op_a, int op_b, int m, int n, int total_k, const void* A, int lda, const void* B,
                            int ldb, void* C, int ldc, const Stack& kg, const char* name, const Call& c) {
  const int tm = (m + 63) / 64;
  dim3 grid((n + 63) / 64, tm < 65535 ? tm : 65535, kg.count);
  const long long a_rs = op_a ? 1 : lda, a_cs = op_a ? lda : 1, b_rs = op_b ? 1 : ldb, b_cs = op_b ? ldb : 1;
  gemm_generic_kgrouped_kernel<InT, OutT><<<grid, 256, 0, c.st>>>(
      kg.offs, kg.count, m, n, total_k, static_cast<const InT*>(A), a_rs, a_cs, static_cast<const InT*>(B), b_rs, b_cs,
      static_cast<OutT*>(C), ldc, kg.sc, c.axpby, c.alpha, c.beta);
  g_launches++;
  t_last_kernel = name;
  return last_launch_status();
}

// C_g = round_out(fma(beta, float(C_g), alpha * op(A)[:, K_g] op(B)[K_g, :])) for g < groups, C_g = C + g * stride_c,
// K_g = [end_{g-1}, end_g) with end_{-1} = 0 and end_g = min(max(offs[g], end_{g-1}), total_k) on the device; an empty
// group stores the k == 0 result of _ex.  Argument rules (all before the device is touched, all by division): those
// of gemm16 for an (m, n, total_k) call; negative sizes, groups or stride_c; groups > kMaxGroups; total_k above
// kMaxTotalK; groups > 1 with C_g overlapping (stride_c < (m - 1) * ldc + n); (groups - 1) * stride_c above 2^60;
// tiles the kernel's int work index cannot count; a null offs with work to do.  groups == 0, m == 0 or n == 0 is a
// no-op.
template <int KIND>
int gemm16_grouped_k(int op_a, int op_b, int m, int n, int total_k, float alpha, const uint16_t* A, int lda,
                     const uint16_t* B, int ldb, const int32_t* offs, int groups, float beta, void* C, int ldc,
                     long long stride_c, int out_type, cudaStream_t st) {
  using K16 = Kind16<KIND>;
  using E = typename K16::E;
  if (groups < 0 || stride_c < 0 || groups > kMaxGroups) return B200_ERR_BAD_ARG;
  if (out_type != B200_OUT_F32 && out_type != K16::OUT16) return B200_ERR_BAD_ARG;
  if ((op_a != B200_OP_N && op_a != B200_OP_T) || (op_b != B200_OP_N && op_b != B200_OP_T)) return B200_ERR_BAD_ARG;
  if (m < 0 || n < 0 || total_k < 0 || total_k > kMaxTotalK) return B200_ERR_BAD_ARG;
  if (groups == 0) return 0;
  int rc = check_args(m, n, total_k, A, lda, B, ldb, C, ldc, op_a, op_b);
  if (rc == 1) return 0;
  if (rc) return rc;
  if (!offs) return B200_ERR_BAD_ARG;
  if (groups > 1) {
    if (stride_c < (long long)(m - 1) * ldc + n) return B200_ERR_BAD_ARG;               // C_g would overlap
    if (stride_c > (1LL << 60) / (groups - 1)) return B200_ERR_BAD_ARG;
  }
  // every group's tiles at the narrowest width, with room for w + gridDim.x, in the kernel's int work index
  const long long tiles1 = ((m + 127LL) / 128) * ((n + 127LL) / 128);                   // < 2^48
  if (tiles1 > 0x3FFFFFFFLL / groups) return B200_ERR_BAD_ARG;
  if ((rc = ensure_device())) return rc;
  Call c{st};
  if (alpha != 1.f || beta != 0.f) { c.axpby = 1; c.alpha = alpha; c.beta = beta; }
  const bool c32 = out_type == B200_OUT_F32;
  const Stack kg{groups, 0, 0, groups > 1 ? stride_c : 0, offs};
  if (total_k == 0 || alpha == 0.f)
    return c32 ? degenerate_batched<float>(m, n, C, ldc, kg, c) : degenerate_batched<E>(m, n, C, ldc, kg, c);
  if (op_a != B200_OP_T || op_b != B200_OP_N || !tma_ok(A, lda, B, ldb, 2)) {
    if (c32)
      return launch_generic_kgrouped<E, float>(op_a, op_b, m, n, total_k, A, lda, B, ldb, C, ldc, kg, K16::kGenericKgrp, c);
    return launch_generic_kgrouped<E, E>(op_a, op_b, m, n, total_k, A, lda, B, ldb, C, ldc, kg, K16::kGenericKgrp, c);
  }
  if (c32) return tc16<KIND, float, false, STACK_KGROUP>(op_a, op_b, m, n, total_k, A, lda, B, ldb, C, ldc, c, &kg);
  return tc16<KIND, typename K16::Out16, false, STACK_KGROUP>(op_a, op_b, m, n, total_k, A, lda, B, ldb, C, ldc, c, &kg);
}

static_assert(ACT_NONE == B200_ACT_NONE && ACT_RELU == B200_ACT_RELU && ACT_GELU == B200_ACT_GELU &&
              ACT_GELU_TANH == B200_ACT_GELU_TANH, "EpiAct follows the header's codes");

// int8 -> int32, C = op(A) op(B).
int gemm_s8(int op_a, int op_b, int m, int n, int k, const int8_t* A, int lda, const int8_t* B, int ldb, int32_t* C,
            int ldc, cudaStream_t st) {
  int rc = check_args(m, n, k, A, lda, B, ldb, C, ldc, op_a, op_b);
  if (rc == 1) return 0;
  if (rc) return rc;
  if ((rc = ensure_device())) return rc;
  Call c{st};
  if (k == 0) return launch_zero<int32_t>(m, n, C, ldc, st);
  if (!tma_ok(A, lda, B, ldb, 1))
    return launch_generic<int8_t, int32_t>(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, "generic_s8_64x64", c);
  return tc_s8(op_a, op_b, m, n, k, A, lda, B, ldb, C, ldc, c);
}

// ---- FP8 (torch._scaled_mm, torch._scaled_grouped_mm) ----------------------------------------------------------------
// Each FP8 entry point describes its call in an Fp8Call, and fp8_gemm checks it (fp8_check) and runs it.
// Kernel names by [stacking][kind][C type: fp32, bf16, fp16, e4m3, e5m2][width index, 3 = promoted, 4 = blockwise].
#define FP8_NAMES(P, S)                                                                                                 \
  {{P "_of32" S "_128x256", P "_of32" S "_128x192", P "_of32" S "_128x128", P "_of32" S "_acc_128x128",                  \
    P "_of32" S "_blk_128x128"},                                                                                         \
   {P "_obf16" S "_128x256", P "_obf16" S "_128x192", P "_obf16" S "_128x128", P "_obf16" S "_acc_128x128",              \
    P "_obf16" S "_blk_128x128"},                                                                                        \
   {P "_of16" S "_128x256", P "_of16" S "_128x192", P "_of16" S "_128x128", P "_of16" S "_acc_128x128",                  \
    P "_of16" S "_blk_128x128"},                                                                                         \
   {P "_oe4m3" S "_128x256", nullptr, P "_oe4m3" S "_128x128", P "_oe4m3" S "_acc_128x128", P "_oe4m3" S "_blk_128x128"}, \
   {P "_oe5m2" S "_128x256", nullptr, P "_oe5m2" S "_128x128", P "_oe5m2" S "_acc_128x128", P "_oe5m2" S "_blk_128x128"}}
const char* const kFp8Names[3][3][5][5] = {
    {FP8_NAMES("tc_e4m3", ""), FP8_NAMES("tc_e4m3e5m2", ""), FP8_NAMES("tc_e5m2e4m3", "")},
    {FP8_NAMES("tc_e4m3", "_bat"), FP8_NAMES("tc_e4m3e5m2", "_bat"), FP8_NAMES("tc_e5m2e4m3", "_bat")},
    {FP8_NAMES("tc_e4m3", "_grp"), FP8_NAMES("tc_e4m3e5m2", "_grp"), FP8_NAMES("tc_e5m2e4m3", "_grp")}};
static_assert(STACK_NONE == 0 && STACK_BATCH == 1 && STACK_GROUP == 2, "kFp8Names is indexed by the stacking");
static_assert(KIND_E4M3E5M2 == KIND_E4M3 + 1 && KIND_E5M2E4M3 == KIND_E4M3 + 2, "kFp8Names rows follow the kinds");

// One FP8 call.  A stacked call (torch._scaled_grouped_mm 2-D x 3-D and 3-D x 3-D) is (N, T): a row-major A (m = total_m
// rows for a grouped call) and every B entry stored n x k (B^T); it has no bias and its rowwise scales are per row and
// per column.
struct Fp8Call {
  Fp8Call(int at, int bt, int m_, int n_, int k_, const uint8_t* a, int la, const uint8_t* b, int lb, void* c, int lc)
      : a_type(at), b_type(bt), m(m_), n(n_), k(k_), A(a), lda(la), B(b), ldb(lb), C(c), ldc(lc) {}
  int a_type, b_type, op_a = B200_OP_N, op_b = B200_OP_T;
  int m, n, k;
  const uint8_t* A; int lda;
  const uint8_t* B; int ldb;
  void* C; int ldc;
  int stack = STACK_NONE, count = 1;                    // STACK_GROUP: groups, stride_b, offs; STACK_BATCH: entries
  long long stride_a = 0, stride_b = 0, stride_c = 0;   // elements between entries
  const int32_t* offs = nullptr;                        // [count] cumulative ends of the groups, on the device
  const float* scale_a = nullptr; const float* scale_b = nullptr;
  bool blockwise = false;
  int a_step = 1, b_step = 1;                           // tensorwise (0) or rowwise (1)
  int a_blk = 1, b_blk = 1;                             // blockwise: 1 x 128 or 128 x 128, with TcBlockScale's strides
  long long sa_row = 0, sa_kb = 0, sb_kb = 0, sb_col = 0;
  long long sa_entry = 0, sb_entry = 0;                 // elements between entries' scales
  const void* bias = nullptr;
  int fast = 0;
  bool q8 = false;                                      // C: out_type (B200_OUT_*), or FP8 (c_type) with its quantisation
  int out_type = B200_OUT_F32, c_type = B200_FP8_E4M3, act = B200_ACT_NONE;
  const float* scale_result = nullptr;
  float* scale_c = nullptr;
  long long sc_row = 0, sc_blk = 0, sc_entry = 0;       // scale_c's strides per row, 128-column block and entry
};

// Element index of the last scale of `count` entries `entry_stride` apart, each (rows - 1) * row_stride + (q - 1) *
// kb_stride long, in 128 bits: the C ABI refuses one whose byte offset does not fit a signed 64-bit integer.
__int128 last_scale_index(long long count, long long entry_stride, long long rows, long long q, long long row_stride,
                          long long kb_stride) {
  return (__int128)(count - 1) * entry_stride + (__int128)(rows - 1) * row_stride +
         (__int128)(q > 0 ? q - 1 : 0) * kb_stride;
}

// Every FP8 call's argument checks, all before the device is touched: < 0 an error, 1 nothing to do, 0 run.  The
// families have always checked in different orders, kept so that every call returns the code it always has: an FP8 C's
// own arguments come first; a single-matrix call checks its sizes and pointers (check_args) before the type pair, a
// stacked call after the type pair and its count.  Stacked calls also refuse (B200_ERR_BAD_ARG) groups > kMaxGroups,
// B_g that overlap (grouped) or entries of C that overlap (batch), an entry stride above 2^60 / (count - 1), more tiles
// than the kernel's int index counts and null offsets, and (B200_ERR_UNSUPPORTED) operands not read in place: FP8 has
// no CUDA-core kernel, and staging every expert's weight would copy all of B.  The last index of each blockwise scale,
// and of a dynamic-mode scale_c, has a byte offset that fits a signed 64-bit integer.
int fp8_check(const Fp8Call& f) {
  auto fp8 = [](int t) { return t == B200_FP8_E4M3 || t == B200_FP8_E5M2; };
  if (f.q8) {
    if (!fp8(f.c_type) || f.act < B200_ACT_NONE || f.act > B200_ACT_GELU_TANH) return B200_ERR_BAD_ARG;
    if ((f.scale_c && (f.scale_result || f.sc_row < 0 || f.sc_blk < 0)) || f.sc_entry < 0) return B200_ERR_BAD_ARG;
  } else if (f.out_type != B200_OUT_F32 && f.out_type != B200_OUT_BF16 && f.out_type != B200_OUT_F16) {
    return B200_ERR_BAD_ARG;
  }
  if (!fp8(f.a_type) || !fp8(f.b_type) || (f.fast != 0 && f.fast != 1)) return B200_ERR_BAD_ARG;
  if ((f.a_step != 0 && f.a_step != 1) || (f.b_step != 0 && f.b_step != 1)) return B200_ERR_BAD_ARG;
  if ((f.a_blk != 1 && f.a_blk != 128) || (f.b_blk != 1 && f.b_blk != 128)) return B200_ERR_BAD_ARG;
  if (f.sa_row < 0 || f.sa_kb < 0 || f.sb_kb < 0 || f.sb_col < 0 || f.sa_entry < 0 || f.sb_entry < 0)
    return B200_ERR_BAD_ARG;
  if (f.count < 0 || f.stride_a < 0 || f.stride_b < 0 || f.stride_c < 0) return B200_ERR_BAD_ARG;
  if (f.stack == STACK_GROUP && f.count > kMaxGroups) return B200_ERR_BAD_ARG;
  const bool stacked = f.stack != STACK_NONE;
  int rc = 0;
  if (!stacked && (rc = check_args(f.m, f.n, f.k, f.A, f.lda, f.B, f.ldb, f.C, f.ldc, f.op_a, f.op_b)) < 0) return rc;
  if (stacked && (f.m < 0 || f.n < 0 || f.k < 0)) return B200_ERR_BAD_ARG;
  if (f.a_type == B200_FP8_E5M2 && f.b_type == B200_FP8_E5M2) return B200_ERR_UNSUPPORTED;
  if (f.a_blk == 128 && f.b_blk == 128) return B200_ERR_UNSUPPORTED;      // not a torch recipe
  if (stacked && f.count == 0) return 1;
  if (stacked) rc = check_args(f.m, f.n, f.k, f.A, f.lda, f.B, f.ldb, f.C, f.ldc, f.op_a, f.op_b);
  if (rc) return rc;
  if (!f.scale_a || !f.scale_b || (f.stack == STACK_GROUP && !f.offs)) return B200_ERR_BAD_ARG;
  const long long qn = (f.n + 127LL) / 128, q = (f.k + 127LL) / 128;
  if (f.count > 1) {
    const long long max_stride = (1LL << 60) / (f.count - 1);
    if (f.stride_a > max_stride || f.stride_b > max_stride || f.stride_c > max_stride || f.sa_entry > max_stride ||
        f.sb_entry > max_stride)
      return B200_ERR_BAD_ARG;
    if (f.stack == STACK_GROUP && f.stride_b < (long long)f.n * f.ldb) return B200_ERR_BAD_ARG;
    if (f.stack == STACK_BATCH && (f.stride_c < (long long)(f.m - 1) * f.ldc + f.n ||
                                   ((f.m + 127LL) / 128) * qn > 0x7FFFFFFFLL / 4 / f.count))    // tiles of one entry < 2^48
      return B200_ERR_BAD_ARG;
  }
  if (f.stack == STACK_GROUP && qn > 0x3FFFFFFFLL / grouped_tile_rows(f.m, f.count)) return B200_ERR_BAD_ARG;
  const __int128 max_index = INT64_MAX / 4;
  if (f.blockwise && (last_scale_index(f.count, f.sa_entry, f.a_blk == 1 ? f.m : (f.m + 127LL) / 128, q, f.sa_row,
                                       f.sa_kb) > max_index ||
                      last_scale_index(f.count, f.sb_entry, f.b_blk == 1 ? f.n : qn, q, f.sb_col, f.sb_kb) > max_index))
    return B200_ERR_BAD_ARG;
  if (stacked && f.k > 0 &&
      (!aligned16(f.A) || !aligned16(f.B) || f.lda % 16 || f.ldb % 16 ||
       (f.count > 1 && (!batch_tma_ok(f.stride_a, f.m, f.lda, 1) || !batch_tma_ok(f.stride_b, f.n, f.ldb, 1)))))
    return B200_ERR_UNSUPPORTED;
  if (f.q8 && (f.scale_c || stacked)) {
    // Dynamic mode: scale_c is row-major (m, q_n) (sc_blk == 1, sc_row >= q_n) or outer-dim-major (sc_row == 1,
    // sc_blk >= m), the stride of an extent-1 dimension being free; anything else could overlap.  A batch's entries,
    // sc_entry apart, do not overlap either.  Static mode (no scale_c) is single-matrix only.
    const bool row_major = (qn == 1 || f.sc_blk == 1) && (f.m == 1 || f.sc_row >= qn);
    const bool col_major = (f.m == 1 || f.sc_row == 1) && (qn == 1 || f.sc_blk >= f.m);
    const __int128 last = last_scale_index(1, 0, f.m, qn, f.sc_row, f.sc_blk);
    if (!f.scale_c || !(row_major || col_major) || last > max_index) return B200_ERR_BAD_ARG;
    if (f.stack == STACK_BATCH && f.count > 1 &&
        (f.sc_entry < last + 1 || f.sc_entry > (1LL << 60) / (f.count - 1) ||
         last_scale_index(f.count, f.sc_entry, f.m, qn, f.sc_row, f.sc_blk) > max_index))
      return B200_ERR_BAD_ARG;
  }
  return 0;
}

// The kernel's argument for the call's scale recipe (BLK), C (Q8) and stacking: TcScale ... TcStackBlockScaleQ8.  A
// stacked one takes the stack (st) in launch_tc.
template <bool BLK, bool Q8, int STACK>
using Fp8Arg = std::conditional_t<
    STACK == STACK_NONE,
    std::conditional_t<BLK, std::conditional_t<Q8, TcBlockScaleQ8, TcBlockScale>, std::conditional_t<Q8, TcScaleQ8, TcScale>>,
    std::conditional_t<BLK, std::conditional_t<Q8, TcStackBlockScaleQ8, TcStackBlockScale>,
                       std::conditional_t<Q8, TcStackScaleQ8, TcStackScale>>>;
template <bool BLK, bool Q8, int STACK>
Fp8Arg<BLK, Q8, STACK> fp8_arg(const Fp8Call& f) {
  Fp8Arg<BLK, Q8, STACK> s{};
  s.a = f.scale_a; s.b = f.scale_b; s.bias = f.bias;
  if constexpr (BLK) {
    s.a_row = f.sa_row; s.a_kb = f.sa_kb; s.b_kb = f.sb_kb; s.b_col = f.sb_col; s.a_blk = f.a_blk; s.b_blk = f.b_blk;
  } else {
    s.a_step = f.a_step; s.b_step = f.b_step;
  }
  if constexpr (STACK != STACK_NONE) { s.a_entry_stride = f.sa_entry; s.b_entry_stride = f.sb_entry; }
  if constexpr (Q8) s.q = TcQ8{f.scale_result, f.scale_c, f.sc_row, f.sc_blk, f.act};
  if constexpr (Q8 && STACK != STACK_NONE) s.sc_entry_stride = f.sc_entry;
  return s;
}

// fast: one accumulator over K at pick_bn's width (a batch counts the tiles of all its entries, a grouped call its
// bound of tile rows); else promoted per 128-element k-block (two 64 x BN fp32 tiles in registers: BN = 128).
// Blockwise scales are always promoted; their indices are logical (row, k-block) / (k-block, column), so staging never
// touches them.  An FP8 C has no 192-wide tile: its 128-column scale blocks must not straddle tiles.
// Every layout and pitch of a single matrix runs on the tensor cores: (N, T) with TMA-able operands is read in place;
// otherwise the operands are made K-major and TMA-able in the workspace (stage_kmajor), which holds the same bytes, so
// every route is bit-identical to the aligned (N, T) call.  A stacked call is read in place (fp8_check).
template <int KIND, typename OutT, int STACK, class Scale>
int tc_fp8(const Fp8Call& f, const Stack& stk, const Scale& sc, const char* const (&names)[5], const Call& c) {
  constexpr bool blk = std::is_base_of<TcBlockScale, Scale>::value;
  const int m = f.m, n = f.n, k = f.k;
  auto run = [&](const void* a, long long la, const void* b, long long lb) {
    if constexpr (!blk)
      if (f.fast) {
        const int bn_m = STACK == STACK_GROUP ? 128 : m;
        const int bn_batch = STACK == STACK_GROUP ? (int)grouped_tile_rows(m, stk.count) : stk.count;
        return with_width<!Fp8Out<OutT>::V>(bn_m, n, [&](auto W) {
          using Wd = decltype(W);
          return launch_tc<KIND, Wd::BN, Wd::STAGES, OutT, ProdSingle, 128, LAYOUT_K, LAYOUT_K, false, STACK>(
              m, n, k, a, la, m, 0, b, lb, n, 0, f.C, f.ldc, names[Wd::idx], c, 0, nullptr, nullptr, &stk, &sc);
        }, bn_batch);
      }
    return launch_tc<KIND, 128, Width<128>::STAGES, OutT, ProdPromoted, 128, LAYOUT_K, LAYOUT_K, false, STACK>(
        m, n, k, a, la, m, 0, b, lb, n, 0, f.C, f.ldc, names[blk ? 4 : 3], c, 128, nullptr, nullptr, &stk, &sc);
  };
  if constexpr (STACK == STACK_NONE) {
    const bool copy_a = !f.op_a && !(aligned16(f.A) && f.lda % 16 == 0);
    const bool copy_b = f.op_b && !(aligned16(f.B) && f.ldb % 16 == 0);
    const int sa = f.op_a || copy_a, sb = f.op_b && !copy_b;      // kmajor_ws_bytes / stage_kmajor's view of the layout
    if (sa || !sb) {
      const void* A = f.A; const void* B = f.B;
      long long lda = f.lda, ldb = f.ldb;
      WsLease ws(kmajor_ws_bytes(sa, sb, m, n, k, 1), c.st);
      if (ws.rc) return ws.rc;
      if (int rc = stage_kmajor<uint8_t>(sa, sb, m, n, k, A, lda, B, ldb, ws.base(), c.st, copy_a, copy_b)) return rc;
      return run(A, lda, B, ldb);
    }
  }
  return run(f.A, f.lda, f.B, f.ldb);
}

// k == 0, FP8 C: the element-wise pass (fp8_q8_k0_kernel), no operand and no input scale read.
template <typename OutT>
int fp8_q8_k0(int m, int n, void* C, int ldc, const void* bias, const TcQ8& q, cudaStream_t st) {
  const long long items = (long long)m * ((n + 127) / 128);
  const int blocks = (int)(items < 4096LL * 128 ? (items + 127) / 128 : 4096);
  fp8_q8_k0_kernel<OutT><<<blocks, 128, 0, st>>>(m, n, static_cast<uint8_t*>(C), ldc,
                                                 static_cast<const uint16_t*>(bias), q);
  g_launches++;
  t_last_kernel = "fp8_q8_k0";
  return last_launch_status();
}

// k == 0, stacked FP8 C: act(+0) quantised and d = 1 over the covered rows / entries (fp8_q8_k0_stacked_kernel), no
// scale read.
template <typename OutT, int STACK>
int fp8_q8_k0_stacked(int m, int n, void* C, int ldc, const Stack& stk, const TcQ8& q, long long sc_entry_stride,
                      cudaStream_t st) {
  const long long items = (STACK == STACK_GROUP ? m : (long long)m * stk.count) * ((n + 127) / 128);
  const int blocks = (int)(items < 4096LL * 128 ? (items + 127) / 128 : 4096);
  fp8_q8_k0_stacked_kernel<OutT, STACK><<<blocks, 128, 0, st>>>(stk.offs, stk.count, m, n, static_cast<uint8_t*>(C), ldc,
                                                                stk.sc, q, sc_entry_stride);
  g_launches++;
  t_last_kernel = STACK == STACK_GROUP ? "fp8_q8_k0_grp" : "fp8_q8_k0_bat";
  return last_launch_status();
}

// Every FP8 call: its checks, then one launch.  A batch of one is the single-matrix (N, T) call: the same kernel, name
// and bits.  k == 0 reads no operand and no scale: C = round_out(+0 + bias_j) (or +0) through the bias pass with beta =
// 0 or the zero fill over the rows or entries the call covers, or an FP8 C's element-wise pass.  Otherwise the type
// pair selects the kind, the C type the kernel's OutT, and the stacking and scale recipe the kernel.
int fp8_gemm(Fp8Call f, void* stream) {
  if (int rc = fp8_check(f)) return rc < 0 ? rc : 0;
  if (f.stack == STACK_BATCH && f.count == 1) f.stack = STACK_NONE;
  if (int rc = ensure_device()) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  Call c{st};
  const Stack stk{f.count, f.stride_a, f.count > 1 ? f.stride_b : 0, f.stride_c, f.offs};
  if (f.k == 0 && f.q8) {
    const TcQ8 q{f.scale_result, f.scale_c, f.sc_row, f.sc_blk, f.act};
    auto k0 = [&](auto out) {
      using O = decltype(out);
      if (f.stack == STACK_GROUP) return fp8_q8_k0_stacked<O, STACK_GROUP>(f.m, f.n, f.C, f.ldc, stk, q, f.sc_entry, st);
      if (f.stack == STACK_BATCH) return fp8_q8_k0_stacked<O, STACK_BATCH>(f.m, f.n, f.C, f.ldc, stk, q, f.sc_entry, st);
      return fp8_q8_k0<O>(f.m, f.n, f.C, f.ldc, f.bias, q, st);
    };
    return f.c_type == B200_FP8_E4M3 ? k0(e4m3_out()) : k0(e5m2_out());
  }
  if (f.k == 0) {
    const bool c32 = f.out_type == B200_OUT_F32;
    if (f.stack == STACK_GROUP)
      return c32 ? degenerate_grouped<float>(f.m, f.n, f.C, f.ldc, stk, c) : degenerate_grouped<uint16_t>(f.m, f.n, f.C, f.ldc, stk, c);
    if (f.stack == STACK_BATCH)
      return c32 ? degenerate_batched<float>(f.m, f.n, f.C, f.ldc, stk, c) : degenerate_batched<uint16_t>(f.m, f.n, f.C, f.ldc, stk, c);
    if (f.bias) { c.bias = f.bias; c.act = ACT_NONE; }
    if (c32) return degenerate<float, float>(f.m, f.n, f.C, f.ldc, c);
    if (f.out_type == B200_OUT_BF16) return degenerate<uint16_t, uint16_t>(f.m, f.n, f.C, f.ldc, c);
    return degenerate<__half, __half>(f.m, f.n, f.C, f.ldc, c);
  }
  const int ci = f.q8 ? 3 + (f.c_type == B200_FP8_E5M2) : f.out_type;      // kFp8Names' C type
  auto launch = [&](auto kind, auto out) {
    constexpr int KIND = decltype(kind)::value;
    using OutT = decltype(out);
    auto stacked = [&](auto stack) {
      constexpr int STACK = decltype(stack)::value;
      constexpr bool Q8 = Fp8Out<OutT>::V;
      const auto& names = kFp8Names[STACK][KIND - KIND_E4M3][ci];
      if (f.blockwise) return tc_fp8<KIND, OutT, STACK>(f, stk, fp8_arg<true, Q8, STACK>(f), names, c);
      return tc_fp8<KIND, OutT, STACK>(f, stk, fp8_arg<false, Q8, STACK>(f), names, c);
    };
    if (f.stack == STACK_GROUP) return stacked(std::integral_constant<int, STACK_GROUP>());
    if (f.stack == STACK_BATCH) return stacked(std::integral_constant<int, STACK_BATCH>());
    return stacked(std::integral_constant<int, STACK_NONE>());
  };
  auto by_c = [&](auto kind) {
    if (ci == 0) return launch(kind, float());
    if (ci == 1) return launch(kind, bf16_out());
    if (ci == 2) return launch(kind, f16_out());
    if (ci == 3) return launch(kind, e4m3_out());
    return launch(kind, e5m2_out());
  };
  if (f.a_type == B200_FP8_E5M2) return by_c(std::integral_constant<int, KIND_E5M2E4M3>());
  if (f.b_type == B200_FP8_E5M2) return by_c(std::integral_constant<int, KIND_E4M3E5M2>());
  return by_c(std::integral_constant<int, KIND_E4M3>());
}

}  // namespace

extern "C" {

const char* b200_gemm_version(void) { return "b200gemm 0.3 (sm_90a; wgmma+TMA)"; }

int b200_gemm_device_ok(void) { return ensure_device(); }

const char* b200_gemm_strerror(int code) {
  switch (code) {
    case B200_OK: return "ok";
    case B200_ERR_BAD_ARG: return "bad argument";
    case B200_ERR_NO_DEVICE: return "no usable sm_90 CUDA device (there is no CPU fallback)";
    case B200_ERR_UNSUPPORTED: return "mode not supported for these operands";
    case B200_ERR_TENSORMAP: return "cuTensorMapEncodeTiled failed";
    case B200_ERR_NCCL: return "NCCL failure (b200_nccl_last_error has the text)";
    default: return code > 0 ? cudaGetErrorString((cudaError_t)code) : "unknown";
  }
}

const char* b200_gemm_last_kernel(void) { return t_last_kernel; }
unsigned long long b200_gemm_launch_count(void) { return g_launches.load(); }
int b200_gemm_default_f32_mode(void) { return resolve_f32_mode(B200_F32_AUTO); }
void b200_gemm_set_default_f32_mode(int mode) {
  if (mode >= 0 && mode != B200_F32_AUTO && mode <= B200_F32_F16X2) g_default_f32_mode.store(mode);
}
void b200_gemm_debug_set_b_desc(int lbo_bytes, int sbo_bytes) { g_dbg_b_lbo = lbo_bytes; g_dbg_b_sbo = sbo_bytes; }
void b200_gemm_debug_set_bn(int bn) { g_force_bn = bn; }
void b200_gemm_debug_set_pdl(int v) { g_pdl = (v & 1) != 0; g_prepass_fork = (v & 2) == 0; }
// The sm_90 kernels have one static tile schedule, no CTA pairs and one epilogue form: these hooks of the
// ABI are accepted and have no effect.
void b200_gemm_debug_set_dynamic_sched(int) {}
void b200_gemm_debug_set_cta_group(int) {}
void b200_gemm_debug_set_split_tail(int on) { g_split_tail = on; }
void b200_gemm_debug_last_schedule(int* tiles, int* split, int* full_tiles, int* ctas) {
  const Schedule& s = t_last_schedule;
  if (tiles) *tiles = s.tiles;
  if (split) *split = s.split;
  if (full_tiles) *full_tiles = s.full_tiles;
  if (ctas) *ctas = s.ctas;
}
void b200_gemm_debug_set_epilogue(int) {}
void b200_gemm_debug_set_group_rows(int rows) { g_group_rows = rows; }
void b200_gemm_debug_set_ffma_variant(int v) { g_ffma_halves = v & 1; g_ffma_fat = v < 0 ? -1 : (v >> 1) & 1; }
void b200_gemm_debug_set_split_chunk(int x3_k, int x2_k) {
  g_split_chunk_k[0] = x3_k < 0 ? kSplitChunkDefault[0] : x3_k;
  g_split_chunk_k[1] = x2_k < 0 ? kSplitChunkDefault[1] : x2_k;
  g_split_chunk_k[2] = x2_k < 0 ? kSplitChunkDefault[2] : x2_k;
}
void b200_gemm_debug_kernel_timing(int enable) { g_ktimer.on = enable != 0; g_ktimer.n = 0; }
int b200_gemm_debug_kernel_time_ms(double* sum_ms) {
  double sum = 0;
  int cnt = 0;
  for (int i = 0; i < g_ktimer.n; i++) {
    float ms = 0.f;
    if (cudaEventSynchronize(g_ktimer.ev[i][1]) == cudaSuccess &&
        cudaEventElapsedTime(&ms, g_ktimer.ev[i][0], g_ktimer.ev[i][1]) == cudaSuccess) { sum += ms; cnt++; }
  }
  cudaGetLastError();
  g_ktimer.n = 0;
  if (sum_ms) *sum_ms = sum;
  return cnt;
}

// Grows the split-precision workspace of the current device up front, so that no later compute call
// synchronises or allocates (first use and growth otherwise do: cudaMalloc of the plane buffers).
int b200_gemm_reserve_workspace(size_t bytes) {
  int rc = ensure_device();
  if (rc) return rc;
  std::lock_guard<std::mutex> wlk(t_ctx->ws_mu);
  return split_ws_reserve(bytes);
}
// The largest workspace the fp32 routes of (op_a, op_b, mode) reserve at this size: over TMA-able operands or not,
// plain or with a general (alpha, beta).  An explicit mode has one route that uses any; AUTO may take several.
size_t b200_gemm_workspace_bytes_op(int op_a, int op_b, int m, int n, int k, int precision_mode) {
  if ((op_a != B200_OP_N && op_a != B200_OP_T) || (op_b != B200_OP_N && op_b != B200_OP_T)) return 0;
  if (m <= 0 || n <= 0 || k <= 0) return 0;
  size_t bytes = 0;
  for (int tma = 0; tma < 2; tma++)
    for (int general = 0; general < 2; general++) {
      const size_t b = f32_route_ws_bytes(f32_route(precision_mode, m, n, k, tma, general), op_a, op_b, m, n, k);
      if (b > bytes) bytes = b;
    }
  return bytes;
}
size_t b200_gemm_workspace_bytes(int m, int n, int k, int precision_mode) {
  return b200_gemm_workspace_bytes_op(B200_OP_N, B200_OP_N, m, n, k, precision_mode);
}

int b200_gemm_f32(int m, int n, int k, const float* dA, int lda, const float* dB, int ldb, float* dC,
                  int ldc, int precision_mode, void* stream) {
  return gemm_f32(B200_OP_N, B200_OP_N, m, n, k, 1.f, dA, lda, dB, ldb, 0.f, dC, ldc, precision_mode, (cudaStream_t)stream);
}

int b200_gemm_f32_acc(int m, int n, int k, const float* dA, int lda, const float* dB, int ldb, float* dC,
                      int ldc, int precision_mode, void* stream) {
  return gemm_f32(B200_OP_N, B200_OP_N, m, n, k, 1.f, dA, lda, dB, ldb, 1.f, dC, ldc, precision_mode, (cudaStream_t)stream);
}

int b200_gemm_f32_ex(int m, int n, int k, float alpha, const float* dA, int lda, const float* dB, int ldb, float beta,
                     float* dC, int ldc, int precision_mode, void* stream) {
  return gemm_f32(B200_OP_N, B200_OP_N, m, n, k, alpha, dA, lda, dB, ldb, beta, dC, ldc, precision_mode, (cudaStream_t)stream);
}

int b200_gemm_f32_op(int op_a, int op_b, int m, int n, int k, float alpha, const float* dA, int lda, const float* dB,
                     int ldb, float beta, float* dC, int ldc, int precision_mode, void* stream) {
  return gemm_f32(op_a, op_b, m, n, k, alpha, dA, lda, dB, ldb, beta, dC, ldc, precision_mode, (cudaStream_t)stream);
}

int b200_gemm_bf16(int m, int n, int k, const uint16_t* dA, int lda, const uint16_t* dB, int ldb,
                   void* dC, int ldc, int out_type, void* stream) {
  return gemm16<KIND_F16>(B200_OP_N, B200_OP_N, m, n, k, 1.f, dA, lda, dB, ldb, 0.f, dC, ldc, out_type, nullptr,
                          B200_ACT_NONE, (cudaStream_t)stream);
}

int b200_gemm_f16(int m, int n, int k, const uint16_t* dA, int lda, const uint16_t* dB, int ldb,
                  void* dC, int ldc, int out_type, void* stream) {
  return gemm16<KIND_FP16>(B200_OP_N, B200_OP_N, m, n, k, 1.f, dA, lda, dB, ldb, 0.f, dC, ldc, out_type, nullptr,
                           B200_ACT_NONE, (cudaStream_t)stream);
}

int b200_gemm_bf16_op(int op_a, int op_b, int m, int n, int k, const uint16_t* dA, int lda, const uint16_t* dB, int ldb,
                      void* dC, int ldc, int out_type, void* stream) {
  return gemm16<KIND_F16>(op_a, op_b, m, n, k, 1.f, dA, lda, dB, ldb, 0.f, dC, ldc, out_type, nullptr, B200_ACT_NONE,
                          (cudaStream_t)stream);
}

int b200_gemm_bf16_ex(int op_a, int op_b, int m, int n, int k, float alpha, const uint16_t* dA, int lda,
                      const uint16_t* dB, int ldb, float beta, void* dC, int ldc, int out_type, void* stream) {
  return gemm16<KIND_F16>(op_a, op_b, m, n, k, alpha, dA, lda, dB, ldb, beta, dC, ldc, out_type, nullptr, B200_ACT_NONE,
                          (cudaStream_t)stream);
}

int b200_gemm_f16_ex(int op_a, int op_b, int m, int n, int k, float alpha, const uint16_t* dA, int lda,
                     const uint16_t* dB, int ldb, float beta, void* dC, int ldc, int out_type, void* stream) {
  return gemm16<KIND_FP16>(op_a, op_b, m, n, k, alpha, dA, lda, dB, ldb, beta, dC, ldc, out_type, nullptr, B200_ACT_NONE,
                           (cudaStream_t)stream);
}

int b200_gemm_bf16_epi(int op_a, int op_b, int m, int n, int k, float alpha, const uint16_t* dA, int lda,
                       const uint16_t* dB, int ldb, float beta, void* dC, int ldc, int out_type, const uint16_t* dBias,
                       int act, void* stream) {
  return gemm16<KIND_F16>(op_a, op_b, m, n, k, alpha, dA, lda, dB, ldb, beta, dC, ldc, out_type, dBias, act,
                          (cudaStream_t)stream);
}

int b200_gemm_f16_epi(int op_a, int op_b, int m, int n, int k, float alpha, const uint16_t* dA, int lda,
                      const uint16_t* dB, int ldb, float beta, void* dC, int ldc, int out_type, const uint16_t* dBias,
                      int act, void* stream) {
  return gemm16<KIND_FP16>(op_a, op_b, m, n, k, alpha, dA, lda, dB, ldb, beta, dC, ldc, out_type, dBias, act,
                           (cudaStream_t)stream);
}

int b200_gemm_bf16_batched(int op_a, int op_b, int m, int n, int k, float alpha, const uint16_t* dA, int lda,
                           long long stride_a, const uint16_t* dB, int ldb, long long stride_b, float beta, void* dC,
                           int ldc, long long stride_c, int batch, int out_type, void* stream) {
  return gemm16_batched<KIND_F16>(op_a, op_b, m, n, k, alpha, dA, lda, stride_a, dB, ldb, stride_b, beta, dC, ldc,
                                  stride_c, batch, out_type, (cudaStream_t)stream);
}

int b200_gemm_f16_batched(int op_a, int op_b, int m, int n, int k, float alpha, const uint16_t* dA, int lda,
                          long long stride_a, const uint16_t* dB, int ldb, long long stride_b, float beta, void* dC,
                          int ldc, long long stride_c, int batch, int out_type, void* stream) {
  return gemm16_batched<KIND_FP16>(op_a, op_b, m, n, k, alpha, dA, lda, stride_a, dB, ldb, stride_b, beta, dC, ldc,
                                   stride_c, batch, out_type, (cudaStream_t)stream);
}

int b200_gemm_bf16_grouped(int op_b, int total_m, int n, int k, float alpha, const uint16_t* dA, int lda,
                           const uint16_t* dB, int ldb, long long stride_b, const int32_t* dOffs, int groups, float beta,
                           void* dC, int ldc, int out_type, void* stream) {
  return gemm16_grouped<KIND_F16>(op_b, total_m, n, k, alpha, dA, lda, dB, ldb, stride_b, dOffs, groups, beta, dC, ldc,
                                  out_type, (cudaStream_t)stream);
}

int b200_gemm_f16_grouped(int op_b, int total_m, int n, int k, float alpha, const uint16_t* dA, int lda,
                          const uint16_t* dB, int ldb, long long stride_b, const int32_t* dOffs, int groups, float beta,
                          void* dC, int ldc, int out_type, void* stream) {
  return gemm16_grouped<KIND_FP16>(op_b, total_m, n, k, alpha, dA, lda, dB, ldb, stride_b, dOffs, groups, beta, dC, ldc,
                                   out_type, (cudaStream_t)stream);
}

int b200_gemm_bf16_grouped_k(int op_a, int op_b, int m, int n, int total_k, float alpha, const uint16_t* dA, int lda,
                             const uint16_t* dB, int ldb, const int32_t* dOffs, int groups, float beta, void* dC,
                             int ldc, long long stride_c, int out_type, void* stream) {
  return gemm16_grouped_k<KIND_F16>(op_a, op_b, m, n, total_k, alpha, dA, lda, dB, ldb, dOffs, groups, beta, dC, ldc,
                                    stride_c, out_type, (cudaStream_t)stream);
}

int b200_gemm_f16_grouped_k(int op_a, int op_b, int m, int n, int total_k, float alpha, const uint16_t* dA, int lda,
                            const uint16_t* dB, int ldb, const int32_t* dOffs, int groups, float beta, void* dC,
                            int ldc, long long stride_c, int out_type, void* stream) {
  return gemm16_grouped_k<KIND_FP16>(op_a, op_b, m, n, total_k, alpha, dA, lda, dB, ldb, dOffs, groups, beta, dC, ldc,
                                     stride_c, out_type, (cudaStream_t)stream);
}

int b200_gemm_s8s32(int m, int n, int k, const int8_t* dA, int lda, const int8_t* dB, int ldb,
                    int32_t* dC, int ldc, void* stream) {
  return gemm_s8(B200_OP_N, B200_OP_N, m, n, k, dA, lda, dB, ldb, dC, ldc, (cudaStream_t)stream);
}

int b200_gemm_fp8(int op_a, int op_b, int a_type, int b_type, int m, int n, int k, const uint8_t* dA, int lda,
                  const uint8_t* dB, int ldb, const float* dScaleA, int scale_a_rowwise, const float* dScaleB,
                  int scale_b_colwise, const void* dBias, void* dC, int ldc, int out_type, int fast_accum, void* stream) {
  Fp8Call f(a_type, b_type, m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.op_a = op_a; f.op_b = op_b;
  f.scale_a = dScaleA; f.a_step = scale_a_rowwise; f.scale_b = dScaleB; f.b_step = scale_b_colwise;
  f.bias = dBias; f.fast = fast_accum; f.out_type = out_type;
  return fp8_gemm(f, stream);
}

int b200_gemm_fp8_blockwise(int op_a, int op_b, int a_type, int b_type, int m, int n, int k, const uint8_t* dA, int lda,
                            const uint8_t* dB, int ldb, const float* dScaleA, int scale_a_block, long long sa_row_stride,
                            long long sa_kb_stride, const float* dScaleB, int scale_b_block, long long sb_kb_stride,
                            long long sb_col_stride, const void* dBias, void* dC, int ldc, int out_type, void* stream) {
  Fp8Call f(a_type, b_type, m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.op_a = op_a; f.op_b = op_b;
  f.blockwise = true;
  f.scale_a = dScaleA; f.a_blk = scale_a_block; f.sa_row = sa_row_stride; f.sa_kb = sa_kb_stride;
  f.scale_b = dScaleB; f.b_blk = scale_b_block; f.sb_kb = sb_kb_stride; f.sb_col = sb_col_stride;
  f.bias = dBias; f.out_type = out_type;
  return fp8_gemm(f, stream);
}

int b200_gemm_fp8_q8(int op_a, int op_b, int a_type, int b_type, int m, int n, int k, const uint8_t* dA, int lda,
                     const uint8_t* dB, int ldb, const float* dScaleA, int scale_a_rowwise, const float* dScaleB,
                     int scale_b_colwise, const uint16_t* dBiasBf16, int act, int fast_accum, int c_type, uint8_t* dC,
                     int ldc, const float* dScaleResult, float* dScaleC, long long sc_row_stride,
                     long long sc_blk_stride, void* stream) {
  Fp8Call f(a_type, b_type, m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.op_a = op_a; f.op_b = op_b;
  f.scale_a = dScaleA; f.a_step = scale_a_rowwise; f.scale_b = dScaleB; f.b_step = scale_b_colwise;
  f.bias = dBiasBf16; f.fast = fast_accum;
  f.q8 = true; f.c_type = c_type; f.act = act; f.scale_result = dScaleResult;
  f.scale_c = dScaleC; f.sc_row = sc_row_stride; f.sc_blk = sc_blk_stride;
  return fp8_gemm(f, stream);
}

int b200_gemm_fp8_blockwise_q8(int op_a, int op_b, int a_type, int b_type, int m, int n, int k, const uint8_t* dA,
                               int lda, const uint8_t* dB, int ldb, const float* dScaleA, int scale_a_block,
                               long long sa_row_stride, long long sa_kb_stride, const float* dScaleB, int scale_b_block,
                               long long sb_kb_stride, long long sb_col_stride, const uint16_t* dBiasBf16, int act,
                               int c_type, uint8_t* dC, int ldc, const float* dScaleResult, float* dScaleC,
                               long long sc_row_stride, long long sc_blk_stride, void* stream) {
  Fp8Call f(a_type, b_type, m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.op_a = op_a; f.op_b = op_b;
  f.blockwise = true;
  f.scale_a = dScaleA; f.a_blk = scale_a_block; f.sa_row = sa_row_stride; f.sa_kb = sa_kb_stride;
  f.scale_b = dScaleB; f.b_blk = scale_b_block; f.sb_kb = sb_kb_stride; f.sb_col = sb_col_stride;
  f.bias = dBiasBf16;
  f.q8 = true; f.c_type = c_type; f.act = act; f.scale_result = dScaleResult;
  f.scale_c = dScaleC; f.sc_row = sc_row_stride; f.sc_blk = sc_blk_stride;
  return fp8_gemm(f, stream);
}

int b200_gemm_fp8_grouped(int a_type, int b_type, int total_m, int n, int k, const uint8_t* dA, int lda,
                          const uint8_t* dB, int ldb, long long stride_b, const int32_t* dOffs, int groups,
                          const float* dScaleA, const float* dScaleB, long long scale_b_stride, void* dC, int ldc,
                          int out_type, int fast_accum, void* stream) {
  Fp8Call f(a_type, b_type, total_m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.stack = STACK_GROUP; f.count = groups; f.stride_b = stride_b; f.offs = dOffs;
  f.scale_a = dScaleA; f.scale_b = dScaleB; f.sb_entry = scale_b_stride;
  f.fast = fast_accum; f.out_type = out_type;
  return fp8_gemm(f, stream);
}

int b200_gemm_fp8_batched(int a_type, int b_type, int m, int n, int k, const uint8_t* dA, int lda, long long stride_a,
                          const uint8_t* dB, int ldb, long long stride_b, const float* dScaleA, long long scale_a_stride,
                          const float* dScaleB, long long scale_b_stride, void* dC, int ldc, long long stride_c,
                          int batch, int out_type, int fast_accum, void* stream) {
  Fp8Call f(a_type, b_type, m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.stack = STACK_BATCH; f.count = batch; f.stride_a = stride_a; f.stride_b = stride_b; f.stride_c = stride_c;
  f.scale_a = dScaleA; f.sa_entry = scale_a_stride; f.scale_b = dScaleB; f.sb_entry = scale_b_stride;
  f.fast = fast_accum; f.out_type = out_type;
  return fp8_gemm(f, stream);
}

int b200_gemm_fp8_blockwise_grouped(int a_type, int b_type, int total_m, int n, int k, const uint8_t* dA, int lda,
                                    const uint8_t* dB, int ldb, long long stride_b, const int32_t* dOffs, int groups,
                                    const float* dScaleA, long long sa_row_stride, long long sa_kb_stride,
                                    const float* dScaleB, int scale_b_block, long long sb_kb_stride,
                                    long long sb_col_stride, long long scale_b_stride, void* dC, int ldc, int out_type,
                                    void* stream) {
  Fp8Call f(a_type, b_type, total_m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.stack = STACK_GROUP; f.count = groups; f.stride_b = stride_b; f.offs = dOffs;
  f.blockwise = true;
  f.scale_a = dScaleA; f.sa_row = sa_row_stride; f.sa_kb = sa_kb_stride;
  f.scale_b = dScaleB; f.b_blk = scale_b_block; f.sb_kb = sb_kb_stride; f.sb_col = sb_col_stride;
  f.sb_entry = scale_b_stride;
  f.out_type = out_type;
  return fp8_gemm(f, stream);
}

int b200_gemm_fp8_blockwise_batched(int a_type, int b_type, int m, int n, int k, const uint8_t* dA, int lda,
                                    long long stride_a, const uint8_t* dB, int ldb, long long stride_b,
                                    const float* dScaleA, int scale_a_block, long long sa_row_stride,
                                    long long sa_kb_stride, long long scale_a_stride, const float* dScaleB,
                                    int scale_b_block, long long sb_kb_stride, long long sb_col_stride,
                                    long long scale_b_stride, void* dC, int ldc, long long stride_c, int batch,
                                    int out_type, void* stream) {
  Fp8Call f(a_type, b_type, m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.stack = STACK_BATCH; f.count = batch; f.stride_a = stride_a; f.stride_b = stride_b; f.stride_c = stride_c;
  f.blockwise = true;
  f.scale_a = dScaleA; f.a_blk = scale_a_block; f.sa_row = sa_row_stride; f.sa_kb = sa_kb_stride;
  f.sa_entry = scale_a_stride;
  f.scale_b = dScaleB; f.b_blk = scale_b_block; f.sb_kb = sb_kb_stride; f.sb_col = sb_col_stride;
  f.sb_entry = scale_b_stride;
  f.out_type = out_type;
  return fp8_gemm(f, stream);
}

int b200_gemm_fp8_grouped_q8(int a_type, int b_type, int total_m, int n, int k, const uint8_t* dA, int lda,
                             const uint8_t* dB, int ldb, long long stride_b, const int32_t* dOffs, int groups,
                             const float* dScaleA, const float* dScaleB, long long scale_b_stride, int act,
                             int fast_accum, int c_type, uint8_t* dC, int ldc, float* dScaleC, long long sc_row_stride,
                             long long sc_blk_stride, void* stream) {
  Fp8Call f(a_type, b_type, total_m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.stack = STACK_GROUP; f.count = groups; f.stride_b = stride_b; f.offs = dOffs;
  f.scale_a = dScaleA; f.scale_b = dScaleB; f.sb_entry = scale_b_stride;
  f.fast = fast_accum;
  f.q8 = true; f.c_type = c_type; f.act = act; f.scale_c = dScaleC; f.sc_row = sc_row_stride; f.sc_blk = sc_blk_stride;
  return fp8_gemm(f, stream);
}

int b200_gemm_fp8_batched_q8(int a_type, int b_type, int m, int n, int k, const uint8_t* dA, int lda, long long stride_a,
                             const uint8_t* dB, int ldb, long long stride_b, const float* dScaleA,
                             long long scale_a_stride, const float* dScaleB, long long scale_b_stride, int act,
                             int fast_accum, int c_type, uint8_t* dC, int ldc, long long stride_c, float* dScaleC,
                             long long sc_row_stride, long long sc_blk_stride, long long sc_entry_stride, int batch,
                             void* stream) {
  Fp8Call f(a_type, b_type, m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.stack = STACK_BATCH; f.count = batch; f.stride_a = stride_a; f.stride_b = stride_b; f.stride_c = stride_c;
  f.scale_a = dScaleA; f.sa_entry = scale_a_stride; f.scale_b = dScaleB; f.sb_entry = scale_b_stride;
  f.fast = fast_accum;
  f.q8 = true; f.c_type = c_type; f.act = act; f.scale_c = dScaleC; f.sc_row = sc_row_stride; f.sc_blk = sc_blk_stride;
  f.sc_entry = sc_entry_stride;
  return fp8_gemm(f, stream);
}

int b200_gemm_fp8_blockwise_grouped_q8(int a_type, int b_type, int total_m, int n, int k, const uint8_t* dA, int lda,
                                       const uint8_t* dB, int ldb, long long stride_b, const int32_t* dOffs, int groups,
                                       const float* dScaleA, long long sa_row_stride, long long sa_kb_stride,
                                       const float* dScaleB, int scale_b_block, long long sb_kb_stride,
                                       long long sb_col_stride, long long scale_b_stride, int act, int c_type,
                                       uint8_t* dC, int ldc, float* dScaleC, long long sc_row_stride,
                                       long long sc_blk_stride, void* stream) {
  Fp8Call f(a_type, b_type, total_m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.stack = STACK_GROUP; f.count = groups; f.stride_b = stride_b; f.offs = dOffs;
  f.blockwise = true;
  f.scale_a = dScaleA; f.sa_row = sa_row_stride; f.sa_kb = sa_kb_stride;
  f.scale_b = dScaleB; f.b_blk = scale_b_block; f.sb_kb = sb_kb_stride; f.sb_col = sb_col_stride;
  f.sb_entry = scale_b_stride;
  f.q8 = true; f.c_type = c_type; f.act = act; f.scale_c = dScaleC; f.sc_row = sc_row_stride; f.sc_blk = sc_blk_stride;
  return fp8_gemm(f, stream);
}

int b200_gemm_fp8_blockwise_batched_q8(int a_type, int b_type, int m, int n, int k, const uint8_t* dA, int lda,
                                       long long stride_a, const uint8_t* dB, int ldb, long long stride_b,
                                       const float* dScaleA, int scale_a_block, long long sa_row_stride,
                                       long long sa_kb_stride, long long scale_a_stride, const float* dScaleB,
                                       int scale_b_block, long long sb_kb_stride, long long sb_col_stride,
                                       long long scale_b_stride, int act, int c_type, uint8_t* dC, int ldc,
                                       long long stride_c, float* dScaleC, long long sc_row_stride,
                                       long long sc_blk_stride, long long sc_entry_stride, int batch, void* stream) {
  Fp8Call f(a_type, b_type, m, n, k, dA, lda, dB, ldb, dC, ldc);
  f.stack = STACK_BATCH; f.count = batch; f.stride_a = stride_a; f.stride_b = stride_b; f.stride_c = stride_c;
  f.blockwise = true;
  f.scale_a = dScaleA; f.a_blk = scale_a_block; f.sa_row = sa_row_stride; f.sa_kb = sa_kb_stride;
  f.sa_entry = scale_a_stride;
  f.scale_b = dScaleB; f.b_blk = scale_b_block; f.sb_kb = sb_kb_stride; f.sb_col = sb_col_stride;
  f.sb_entry = scale_b_stride;
  f.q8 = true; f.c_type = c_type; f.act = act; f.scale_c = dScaleC; f.sc_row = sc_row_stride; f.sc_blk = sc_blk_stride;
  f.sc_entry = sc_entry_stride;
  return fp8_gemm(f, stream);
}

int b200_gemm_s8s32_op(int op_a, int op_b, int m, int n, int k, const int8_t* dA, int lda, const int8_t* dB, int ldb,
                       int32_t* dC, int ldc, void* stream) {
  return gemm_s8(op_a, op_b, m, n, k, dA, lda, dB, ldb, dC, ldc, (cudaStream_t)stream);
}

// ---- pre-split operands (the reference's "packAB interface is open" idea, README.md:85, for the split modes) ----
// One handle type for both sides: bf16 planes (BF16X3 / BF16X2, B only) or scaled fp16 planes with the
// maxima their scaling came from (F16X2, A or B).
struct b200_packed {
  int side;            // 0 = A (rows x cols = m x k), 1 = B (k x n)
  int rows, cols, mode, np, plane_rows;
  long long pitch;
  uint16_t* planes;
  float* maxv;         // F16X2 only
  int dev;
};
struct b200_packed_a : b200_packed {};
struct b200_packed_b : b200_packed {};

static int pack_operand(int side, int rows, int cols, const float* d, int ld, int precision_mode, b200_packed* h,
                        cudaStream_t st) {
  if (rows <= 0 || cols <= 0 || !d || ld < cols) return B200_ERR_BAD_ARG;
  const int mode = resolve_f32_mode(precision_mode);
  if (mode != B200_F32_F16X2 && (side != 1 || (mode != B200_F32_BF16X3 && mode != B200_F32_BF16X2))) return B200_ERR_UNSUPPORTED;
  int rc = ensure_device();
  if (rc) return rc;
  const PlaneGeom g = side == 0 ? geom_a(B200_OP_N, rows, cols) : geom_b(B200_OP_N, rows, cols);
  h->side = side; h->rows = rows; h->cols = cols; h->mode = mode; h->planes = nullptr; h->maxv = nullptr;
  h->dev = t_ctx->dev;
  h->np = mode == B200_F32_BF16X3 ? 3 : 2;
  h->pitch = g.pitch;
  h->plane_rows = g.plane_rows;
  if (mode == B200_F32_F16X2) {
    const size_t nmax = side == 0 ? (size_t)rows : (size_t)cols;
    cudaError_t e = cudaMalloc(&h->planes, g.bytes(2));
    if (e == cudaSuccess) e = cudaMalloc(&h->maxv, nmax * 4);
    if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
    if (side == 0) return launch_f16_split_rows(d, ld, rows, cols, h->maxv, h->planes, h->pitch, h->plane_rows, st);
    e = cudaMemsetAsync(h->maxv, 0, nmax * 4, st);
    if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
    return launch_f16_split_cols(d, ld, rows, cols, h->maxv, h->planes, h->pitch, h->plane_rows, nullptr, 0, st);
  }
  cudaError_t e = cudaMalloc(&h->planes, g.bytes(h->np));
  if (e != cudaSuccess) { cudaGetLastError(); return (int)e; }
  const SplitJob jb{d, ld, rows, cols, h->planes, h->pitch, h->plane_rows};
  return h->np == 3 ? launch_split<3>(jb, jb, 1, st) : launch_split<2>(jb, jb, 1, st);
}
extern "C++" {
template <class H>
static void pack_destroy(H* h) {
  if (!h) return;
  if (h->planes) cudaFree(h->planes);
  if (h->maxv) cudaFree(h->maxv);
  delete h;
}
template <class H>
static int pack(int side, int rows, int cols, const float* d, int ld, int precision_mode, H** out, cudaStream_t st) {
  if (!out) return B200_ERR_BAD_ARG;
  *out = nullptr;
  H* h = new H();
  int rc = pack_operand(side, rows, cols, d, ld, precision_mode, h, st);
  t_last_kernel = "split_planes";
  if (rc) { pack_destroy(h); return rc; }
  *out = h;
  return B200_OK;
}
}  // extern "C++"

int b200_gemm_f32_pack_b(int k, int n, const float* dB, int ldb, int precision_mode, b200_packed_b** out,
                         void* stream) {
  return pack(1, k, n, dB, ldb, precision_mode, out, (cudaStream_t)stream);
}

int b200_gemm_f32_pack_a(int m, int k, const float* dA, int lda, int precision_mode, b200_packed_a** out,
                         void* stream) {
  return pack(0, m, k, dA, lda, precision_mode, out, (cudaStream_t)stream);
}

// k0: first column of packed A / first row of B this product starts at (K-sliced consumers); the B handle
// always covers exactly the k rows multiplied.
static int gemm_packed_impl(int m, int n, int k, const float* dA, int lda, const b200_packed* pa, int a_k0,
                            const b200_packed* pb, float* dC, int ldc, int accumulate, cudaStream_t st) {
  if (!pb || pb->rows != k || pb->cols != n) return B200_ERR_BAD_ARG;
  if (pa && (pa->rows != m || a_k0 < 0 || a_k0 + k > pa->cols || (a_k0 & 7) || pa->mode != pb->mode)) return B200_ERR_BAD_ARG;
  int rc = check_args(m, n, k, pa ? (const void*)pa->planes : (const void*)dA, pa ? k : lda, pb->planes, n, dC, ldc);
  if (rc == 1) return 0;
  if (rc) return rc;
  rc = ensure_device();
  if (rc) return rc;
  if (pb->dev != t_ctx->dev || (pa && pa->dev != t_ctx->dev)) return B200_ERR_BAD_ARG;
  Call c{st};
  c.acc = accumulate ? 1 : 0;
  const int N = B200_OP_N;
  if (pb->mode == B200_F32_F16X2) {
    const F16Operand ob{pb->planes, pb->pitch, pb->plane_rows, pb->maxv};
    if (pa) {
      const F16Operand oa{pa->planes + a_k0, pa->pitch, pa->plane_rows, pa->maxv};
      return gemm_f32_split_f16(N, N, m, n, k, nullptr, 0, nullptr, 0, dC, ldc, &oa, &ob, c);
    }
    return gemm_f32_split_f16(N, N, m, n, k, dA, lda, nullptr, 0, dC, ldc, nullptr, &ob, c);
  }
  if (pa) return B200_ERR_UNSUPPORTED;
  return pb->np == 3 ? gemm_f32_split<3>(N, N, m, n, k, dA, lda, nullptr, 0, dC, ldc, pb->planes, c)
                     : gemm_f32_split<2>(N, N, m, n, k, dA, lda, nullptr, 0, dC, ldc, pb->planes, c);
}

int b200_gemm_f32_packed(int m, int n, int k, const float* dA, int lda, const b200_packed_b* pb, float* dC,
                         int ldc, int accumulate, void* stream) {
  return gemm_packed_impl(m, n, k, dA, lda, nullptr, 0, pb, dC, ldc, accumulate, (cudaStream_t)stream);
}

int b200_gemm_f32_packed_ab(int m, int n, int k, const b200_packed_a* pa, int a_k0, const b200_packed_b* pb,
                            float* dC, int ldc, int accumulate, void* stream) {
  if (!pa) return B200_ERR_BAD_ARG;
  return gemm_packed_impl(m, n, k, nullptr, 0, pa, a_k0, pb, dC, ldc, accumulate, (cudaStream_t)stream);
}

void b200_gemm_f32_pack_free(b200_packed_b* pb) { pack_destroy(pb); }
void b200_gemm_f32_pack_free_a(b200_packed_a* pa) { pack_destroy(pa); }

int b200_gemm_s8s8_requant(int m, int n, int k, const int8_t* dA, int lda, const int8_t* dB, int ldb,
                           int8_t* dC, int ldc, const float* dScales, const float* dBias, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  int rc = check_args(m, n, k, dA, lda, dB, ldb, dC, ldc);
  if (rc == 1) return 0;
  if (rc) return rc;
  if (!dScales) return B200_ERR_BAD_ARG;
  rc = ensure_device();
  if (rc) return rc;
  if (k == 0 || !tma_ok(dA, lda, dB, ldb, 1))         // K = 0: every element is requant(0) = sat(round(bias))
    return launch_generic_requant(m, n, k, dA, lda, dB, ldb, dC, ldc, dScales, dBias, st);
  Call c{st};
  return tc_s8_requant(m, n, k, dA, lda, dB, ldb, dC, ldc, dScales, dBias, c);
}

// ---- the 4-bit path: block-scaled MXFP4 (SURVEY §8 f-4; the reference's cuda-int4 is "WIP") ----------------
size_t b200_mxf4_q_bytes(int rows, int k) { return rows <= 0 || k <= 0 ? 0 : (size_t)rows * (size_t)(((k + 127) & ~127) / 2); }
size_t b200_mxf4_sf_bytes(int rows, int k) {
  return rows <= 0 || k <= 0 ? 0 : (size_t)((rows + 127) / 128) * (size_t)((k + 127) / 128) * 512;
}

int b200_mxf4_quantize_a(int m, int k, const float* dA, int lda, uint8_t* dQ, uint8_t* dSF, void* stream) {
  if (m <= 0 || k <= 0 || !dA || !dQ || !dSF || lda < k) return B200_ERR_BAD_ARG;
  int rc = ensure_device();
  if (rc) return rc;
  const int kpad = (k + 127) & ~127, rows_pad = (m + 127) & ~127;
  const long long total = (long long)rows_pad * (kpad / 32);
  long long blocks = (total + 255) / 256;
  if (blocks > t_ctx->sms * 16) blocks = t_ctx->sms * 16;
  mxf4_quantize_rows_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(dA, lda, m, k, dQ, kpad, dSF, rows_pad);
  g_launches++;
  t_last_kernel = "mxf4_quantize_rows";
  return last_launch_status();
}

// B is k x n row-major; the output is B^T quantised along K: n rows of kpad/2 bytes (the K-major operand the
// 4-bit tensor path requires) + scale atoms indexed by (n, K-block).
int b200_mxf4_quantize_b(int k, int n, const float* dB, int ldb, uint8_t* dQ, uint8_t* dSF, void* stream) {
  if (n <= 0 || k <= 0 || !dB || !dQ || !dSF || ldb < n) return B200_ERR_BAD_ARG;
  int rc = ensure_device();
  if (rc) return rc;
  const int kpad = (k + 127) & ~127, n_pad = (n + 127) & ~127;
  mxf4_quantize_cols_t_kernel<<<dim3((n_pad + 255) / 256, grid_y(kpad / 32)), 256, 0, (cudaStream_t)stream>>>(dB, ldb, k, n, dQ, kpad, dSF, n_pad);
  g_launches++;
  t_last_kernel = "mxf4_quantize_cols_t";
  return last_launch_status();
}

int b200_gemm_mxf4(int m, int n, int k, const uint8_t* dAq, const uint8_t* dSFA, const uint8_t* dBq, const uint8_t* dSFB,
                   float* dC, int ldc, void* stream) {
  if (m < 0 || n < 0 || k < 0) return B200_ERR_BAD_ARG;
  if (m == 0 || n == 0) return 0;
  if (!dC || ldc < n) return B200_ERR_BAD_ARG;
  int rc = ensure_device();
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (k == 0) return launch_zero<float>(m, n, dC, ldc, st);
  if (!dAq || !dSFA || !dBq || !dSFB || !aligned16(dAq) || !aligned16(dBq) || !aligned16(dSFA) || !aligned16(dSFB)) return B200_ERR_BAD_ARG;
  // both operands expanded (exactly) to bf16 in the workspace, then the bf16 tensor-core GEMM (gemm_mxf4.cuh)
  const int kpad = (k + 127) & ~127;
  const long long npitch = ((long long)n + 7) & ~7LL;
  const size_t a_bytes = ((size_t)m * kpad * 2 + 1023) & ~(size_t)1023;
  WsLease ws(a_bytes + (size_t)kpad * npitch * 2, st);
  if (ws.rc) return ws.rc;
  uint16_t* a16 = reinterpret_cast<uint16_t*>(ws.base());
  uint16_t* b16 = reinterpret_cast<uint16_t*>(ws.base() + a_bytes);
  long long blocks = ((long long)m * (kpad / 32) + 255) / 256;
  if (blocks > t_ctx->sms * 16) blocks = t_ctx->sms * 16;
  launch_pdl(mxf4_expand_rows_kernel, dim3((unsigned)blocks), dim3(256), 0, st, 1, dAq, dSFA, m, kpad, a16);
  launch_pdl(mxf4_expand_cols_t_kernel, dim3((n + 255) / 256, grid_y(kpad / 32)), dim3(256), 0, st, 1, dBq, dSFB, n, kpad, b16, npitch);
  g_launches += 2;
  if ((rc = last_launch_status())) return rc;
  Call c{st};
  return launch_tc<KIND_F16, 128, 6, float>(m, n, kpad, a16, kpad, m, 0, b16, npitch, kpad, 0, dC, ldc, "tc_mxf4_128x128", c);
}

// ---- blockwise FP8 quantisers (fp8_quant.cuh): the producers of b200_gemm_fp8_blockwise's operands ----------------
extern "C++" {
namespace {
// The layout rule of b200_gemm_fp8_q8's dScaleC over (rows, blks): row-major or outer-dim-major, the stride of an
// extent-1 dimension being free.
bool scale_layout_ok(long long rows, long long blks, long long s_row, long long s_blk) {
  const bool row_major = (blks == 1 || s_blk == 1) && (rows == 1 || s_row >= blks);
  const bool col_major = (rows == 1 || s_row == 1) && (blks == 1 || s_blk >= rows);
  return row_major || col_major;
}

template <typename In, typename OutT, int BLK, bool TRANS>
int launch_fp8_quant(const Fp8QuantArgs& a, cudaStream_t st) {
  auto kern = fp8_quant_kernel<In, OutT, BLK, TRANS>;
  const int smem = TRANS ? quant_smem_bytes<In>() : 0;
  int rc = smem > 48 * 1024 ? ensure_smem_attr(kern, smem) : 0;
  if (rc) return rc;
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kQuantThreads, smem) != cudaSuccess || per_sm < 1) {
    cudaGetLastError();
    per_sm = 1;
  }
  const long long cap = (long long)t_ctx->sms * per_sm;
  kern<<<(unsigned)(a.tiles < cap ? a.tiles : cap), kQuantThreads, smem, st>>>(a);
  return 0;
}

template <typename In, typename OutT>
int fp8_quant_recipe(const Fp8QuantArgs& a, int block, const char* const (&names)[4], cudaStream_t st) {
  const int i = (block == 128 ? 2 : 0) + (a.qt ? 1 : 0);
  t_last_kernel = names[i];
  switch (i) {
    case 0: return launch_fp8_quant<In, OutT, 1, false>(a, st);
    case 1: return launch_fp8_quant<In, OutT, 1, true>(a, st);
    case 2: return launch_fp8_quant<In, OutT, 128, false>(a, st);
    default: return launch_fp8_quant<In, OutT, 128, true>(a, st);
  }
}

template <typename In>
int fp8_quant_in(const Fp8QuantArgs& a, int c_type, int block, const char* const (&e4)[4], const char* const (&e5)[4],
                 cudaStream_t st) {
  return c_type == B200_FP8_E4M3 ? fp8_quant_recipe<In, e4m3_out>(a, block, e4, st)
                                 : fp8_quant_recipe<In, e5m2_out>(a, block, e5, st);
}
}  // namespace
}  // extern "C++"

int b200_fp8_quantize(int in_type, int c_type, int block, int rows, int cols, int batch,
                      const void* dX, int ldx, long long stride_x,
                      uint8_t* dQ, int ldq, long long stride_q,
                      float* dScale, long long s_row, long long s_blk, long long s_entry,
                      uint8_t* dQt, int ldqt, long long stride_qt,
                      float* dScaleT, long long st_row, long long st_blk, long long st_entry, void* stream) {
  if (in_type != B200_OUT_F32 && in_type != B200_OUT_BF16 && in_type != B200_OUT_F16) return B200_ERR_BAD_ARG;
  if ((c_type != B200_FP8_E4M3 && c_type != B200_FP8_E5M2) || (block != 1 && block != 128)) return B200_ERR_BAD_ARG;
  if (rows < 0 || cols < 0 || batch < 0 || stride_x < 0 || stride_q < 0 || s_row < 0 || s_blk < 0 || s_entry < 0 ||
      stride_qt < 0 || st_row < 0 || st_blk < 0 || st_entry < 0)
    return B200_ERR_BAD_ARG;
  if (rows == 0 || cols == 0 || batch == 0) return 0;
  const bool trans = dQt != nullptr;
  if (ldx < cols || ldq < cols || (trans && ldqt < rows)) return B200_ERR_BAD_ARG;
  if (!dX || !dQ || !dScale || (block == 1 && trans != (dScaleT != nullptr)) || (block == 128 && dScaleT))
    return B200_ERR_BAD_ARG;
  // scales: (rows, qc) for 1 x 128, (qr, qc) for 128 x 128; the transposed output's (cols, qr) for 1 x 128
  const long long qr = (rows + 127LL) / 128, qc = (cols + 127LL) / 128, srows = block == 1 ? rows : qr;
  if (!scale_layout_ok(srows, qc, s_row, s_blk) || (dScaleT && !scale_layout_ok(cols, qr, st_row, st_blk)))
    return B200_ERR_BAD_ARG;
  // batch entries of the outputs must not overlap; strides bounded as the stacked GEMMs' are
  const long long in_bytes = in_type == B200_OUT_F32 ? 4 : 2;
  const long long q_last = (rows - 1LL) * ldq + cols - 1, qt_last = trans ? (cols - 1LL) * ldqt + rows - 1 : 0;
  const __int128 s_last = last_scale_index(1, 0, srows, qc, s_row, s_blk);
  const __int128 st_last = dScaleT ? last_scale_index(1, 0, cols, qr, st_row, st_blk) : 0;
  if (batch > 1) {
    const long long max_stride = (1LL << 60) / (batch - 1);
    if (stride_x > max_stride || stride_q > max_stride || s_entry > max_stride || stride_qt > max_stride ||
        st_entry > max_stride)
      return B200_ERR_BAD_ARG;
    if (stride_q <= q_last || s_entry <= s_last || (trans && stride_qt <= qt_last) || (dScaleT && st_entry <= st_last))
      return B200_ERR_BAD_ARG;
  }
  // the last element of every tensor has a byte offset that fits a signed 64-bit integer
  const __int128 e_last = batch - 1;
  if ((e_last * stride_x + (__int128)(rows - 1) * ldx + cols - 1) * in_bytes > INT64_MAX ||
      e_last * stride_q + q_last > INT64_MAX || (e_last * s_entry + s_last) * 4 > INT64_MAX ||
      (trans && e_last * stride_qt + qt_last > INT64_MAX) || (dScaleT && (e_last * st_entry + st_last) * 4 > INT64_MAX))
    return B200_ERR_BAD_ARG;
  int rc = ensure_device();
  if (rc) return rc;
  Fp8QuantArgs a{dX, ldx, batch > 1 ? stride_x : 0, dQ, ldq, batch > 1 ? stride_q : 0, dScale, s_row, s_blk,
                 batch > 1 ? s_entry : 0, dQt, ldqt, batch > 1 ? stride_qt : 0, dScaleT, st_row, st_blk,
                 batch > 1 ? st_entry : 0, rows, cols, (int)qc, qr * qc, qr * qc * batch, 0};
  a.vec = aligned16(dX) && (ldx * in_bytes) % 16 == 0 && (batch == 1 || (stride_x * in_bytes) % 16 == 0);
  cudaStream_t st = (cudaStream_t)stream;
  static const char* const bf16_e4[4] = {"fp8_quant_bf16_e4m3_1x128", "fp8_quant_t_bf16_e4m3_1x128",
                                         "fp8_quant_bf16_e4m3_128x128", "fp8_quant_t_bf16_e4m3_128x128"};
  static const char* const bf16_e5[4] = {"fp8_quant_bf16_e5m2_1x128", "fp8_quant_t_bf16_e5m2_1x128",
                                         "fp8_quant_bf16_e5m2_128x128", "fp8_quant_t_bf16_e5m2_128x128"};
  static const char* const f16_e4[4] = {"fp8_quant_f16_e4m3_1x128", "fp8_quant_t_f16_e4m3_1x128",
                                        "fp8_quant_f16_e4m3_128x128", "fp8_quant_t_f16_e4m3_128x128"};
  static const char* const f16_e5[4] = {"fp8_quant_f16_e5m2_1x128", "fp8_quant_t_f16_e5m2_1x128",
                                        "fp8_quant_f16_e5m2_128x128", "fp8_quant_t_f16_e5m2_128x128"};
  static const char* const f32_e4[4] = {"fp8_quant_f32_e4m3_1x128", "fp8_quant_t_f32_e4m3_1x128",
                                        "fp8_quant_f32_e4m3_128x128", "fp8_quant_t_f32_e4m3_128x128"};
  static const char* const f32_e5[4] = {"fp8_quant_f32_e5m2_1x128", "fp8_quant_t_f32_e5m2_1x128",
                                        "fp8_quant_f32_e5m2_128x128", "fp8_quant_t_f32_e5m2_128x128"};
  if (in_type == B200_OUT_BF16) rc = fp8_quant_in<qin_bf16>(a, c_type, block, bf16_e4, bf16_e5, st);
  else if (in_type == B200_OUT_F16) rc = fp8_quant_in<qin_f16>(a, c_type, block, f16_e4, f16_e5, st);
  else rc = fp8_quant_in<qin_f32>(a, c_type, block, f32_e4, f32_e5, st);
  if (rc) return rc;
  g_launches++;
  return last_launch_status();
}

int b200_convert_f32_to_bf16(const float* dSrc, uint16_t* dDst, size_t count, void* stream) {
  if (count == 0) return 0;
  if (!dSrc || !dDst) return B200_ERR_BAD_ARG;
  int rc = ensure_device();
  if (rc) return rc;
  size_t blocks = (count + 255) / 256;
  if (blocks > (size_t)t_ctx->sms * 32) blocks = (size_t)t_ctx->sms * 32;
  convert_f32_to_bf16_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(dSrc, dDst, count);
  g_launches++;
  t_last_kernel = "convert_f32_to_bf16";
  return last_launch_status();
}

// ---- host-pointer entry points (plumbing / parity / e2e) ---------------------------------------
// Device staging buffers are cached and only ever grow, so repeated calls (the harness calls
// MY_MMult NREPEATS times, aarch64/test_MMult.cpp:105-117) pay no cudaMalloc after the first.
// Copies are asynchronous on the legacy stream; pinned host buffers run at full PCIe rate.
namespace {
cudaError_t scratch(int i, size_t bytes, void** out) {
  Scratch* scr = t_ctx->scr;
  if (scr[i].bytes < bytes) {
    if (scr[i].p) cudaFree(scr[i].p);
    scr[i].p = nullptr; scr[i].bytes = 0;
    cudaError_t e = cudaMalloc(&scr[i].p, bytes);
    if (e != cudaSuccess) return e;
    scr[i].bytes = bytes;
  }
  *out = scr[i].p;
  return cudaSuccess;
}
}  // namespace

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { cudaGetLastError(); return (int)e_; } } while (0)

int b200_gemm_f32_host(int m, int n, int k, const float* A, int lda, const float* B, int ldb, float* C,
                       int ldc, int precision_mode) {
  int rc = check_args(m, n, k, A, lda, B, ldb, C, ldc);
  if (rc == 1) return 0;
  if (rc) return rc;
  rc = ensure_device();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(t_ctx->host_mu);
  float *dA = nullptr, *dB = nullptr, *dC = nullptr;
  const int mode = precision_mode;   // unresolved: AUTO keeps its small-problem switch to the bit-exact STRICT kernel
  // device images: pitches rounded up to 4 floats so the TMA paths apply to any k, n
  const int pk = (k + 3) & ~3, pn = (n + 3) & ~3;
  const size_t pa = (size_t)pk * 4, pb = (size_t)pn * 4, pc = (size_t)pn * 4;
  if (k > 0) {
    CK(scratch(0, pa * m, (void**)&dA));
    CK(scratch(1, pb * k, (void**)&dB));
  }
  CK(scratch(2, pc * m, (void**)&dC));
  // Large problems: row-block pipeline over three streams, so the D2H of C block i overlaps the H2D
  // of block i+1 (PCIe is full duplex) and the GEMMs hide under the copies.  The path is copy-bound:
  // 268 MB cross the bus per 4096^3 call against 0.6 ms of math.
  const int blocks = (k > 0 && m >= 2048 && (double)m * n * k >= 8.0e9) ? 4 : 1;
  if (blocks == 1) {
    cudaStream_t st = 0;
    if (k > 0) {
      CK(cudaMemcpy2DAsync(dA, pa, A, (size_t)lda * 4, (size_t)k * 4, m, cudaMemcpyHostToDevice, st));
      CK(cudaMemcpy2DAsync(dB, pb, B, (size_t)ldb * 4, (size_t)n * 4, k, cudaMemcpyHostToDevice, st));
    }
    CK(cudaMemcpy2DAsync(dC, pc, C, (size_t)ldc * 4, (size_t)n * 4, m, cudaMemcpyHostToDevice, st));
    rc = gemm_f32(B200_OP_N, B200_OP_N, m, n, k, 1.f, dA, pk, dB, pn, 1.f, dC, pn, mode, st);   // C += A*B on the device
    if (rc) return rc;
    CK(cudaMemcpy2DAsync(C, (size_t)ldc * 4, dC, pc, (size_t)n * 4, m, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return 0;
  }
  CK(t_ctx->pipe.init());
  CK(cudaMemcpy2DAsync(dB, pb, B, (size_t)ldb * 4, (size_t)n * 4, k, cudaMemcpyHostToDevice, t_ctx->pipe.h2d));
  const int rows_per = ((m + blocks - 1) / blocks + 255) & ~255;       // whole 256-row pair tiles per block
  int nb = 0;
  for (int r0 = 0; r0 < m; r0 += rows_per, nb++) {
    const int rows = m - r0 < rows_per ? m - r0 : rows_per;
    float* dAi = dA + (size_t)r0 * pk;
    float* dCi = dC + (size_t)r0 * pn;
    CK(cudaMemcpy2DAsync(dAi, pa, A + (size_t)r0 * lda, (size_t)lda * 4, (size_t)k * 4, rows, cudaMemcpyHostToDevice, t_ctx->pipe.h2d));
    CK(cudaMemcpy2DAsync(dCi, pc, C + (size_t)r0 * ldc, (size_t)ldc * 4, (size_t)n * 4, rows, cudaMemcpyHostToDevice, t_ctx->pipe.h2d));
    CK(cudaEventRecord(t_ctx->pipe.in[nb], t_ctx->pipe.h2d));
    CK(cudaStreamWaitEvent(t_ctx->pipe.comp, t_ctx->pipe.in[nb], 0));
    rc = gemm_f32(B200_OP_N, B200_OP_N, rows, n, k, 1.f, dAi, pk, dB, pn, 1.f, dCi, pn, mode, t_ctx->pipe.comp);
    if (rc) return rc;
    CK(cudaEventRecord(t_ctx->pipe.done[nb], t_ctx->pipe.comp));
    CK(cudaStreamWaitEvent(t_ctx->pipe.d2h, t_ctx->pipe.done[nb], 0));
    CK(cudaMemcpy2DAsync(C + (size_t)r0 * ldc, (size_t)ldc * 4, dCi, pc, (size_t)n * 4, rows, cudaMemcpyDeviceToHost, t_ctx->pipe.d2h));
  }
  CK(cudaStreamSynchronize(t_ctx->pipe.d2h));
  CK(cudaStreamSynchronize(t_ctx->pipe.comp));
  return 0;
}

int b200_gemm_s8s32_host(int m, int n, int k, const int8_t* A, int lda, const int8_t* B, int ldb,
                         int32_t* C, int ldc) {
  int rc = check_args(m, n, k, A, lda, B, ldb, C, ldc);
  if (rc == 1) return 0;
  if (rc) return rc;
  rc = ensure_device();
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(t_ctx->host_mu);
  int8_t *dA = nullptr, *dB = nullptr;
  int32_t* dC = nullptr;
  // device images padded to 16-byte pitches so the tensor-core path is taken for any m,n,k
  const size_t pa = ((size_t)k + 15) & ~(size_t)15, pb = ((size_t)n + 15) & ~(size_t)15;
  const size_t pc = (size_t)n * 4;
  cudaStream_t st = 0;
  if (k > 0) {
    CK(scratch(0, pa * m, (void**)&dA));
    CK(scratch(1, pb * k, (void**)&dB));
    CK(cudaMemcpy2DAsync(dA, pa, A, (size_t)lda, (size_t)k, m, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpy2DAsync(dB, pb, B, (size_t)ldb, (size_t)n, k, cudaMemcpyHostToDevice, st));
  }
  CK(scratch(2, pc * m, (void**)&dC));
  rc = b200_gemm_s8s32(m, n, k, dA, (int)pa, dB, (int)pb, dC, n, st);
  if (rc) return rc;
  CK(cudaMemcpy2DAsync(C, (size_t)ldc * 4, dC, pc, pc, m, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"

#include "rowpanel.cuh"
