// rowpanel.cuh — the multi-GPU entry points of the C ABI (included by capi.cu, inside its TU).
//
// Rows of C are independent (SURVEY §8e): rank i owns A_i (m_local x k) and C_i (m_local x n); B (k x n)
// lives on `root` and crosses NVLink once per product, as contiguous row blocks (K-slices) of the
// row-major operand, broadcast in place with ncclBroadcast on a side stream.  The math hides the exchange:
//   * A_i is split into its fp16 planes while the first slice of B is in flight (A never depends on B),
//   * slice j of B is split and multiplied (C_i (+)= A_i[:, ks] * B[ks, :]) while slices j+1.. travel.
// The reference has no multi-GPU code; the timing convention followed is its harness's (operands resident,
// the exchange inside the timed call — cuda/test_MMult.cpp:84-112).
//
// NCCL is resolved at run time (dlopen of the libnccl.so.2 already in the process — torch's — or the system
// one): libb200gemm.so has no link-time dependency on it and loads on boxes without NCCL.
#pragma once
#include <dlfcn.h>
#include <nccl.h>

namespace {

struct NcclApi {
  void* lib = nullptr;
  bool ok = false;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*CommCount)(const ncclComm_t, int*) = nullptr;
  ncclResult_t (*CommUserRank)(const ncclComm_t, int*) = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
} g_nccl;
thread_local char t_nccl_err[256] = "";

int nccl_load(const char* path) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_nccl.ok) return 0;
  const char* names[3] = {path, "libnccl.so.2", "libnccl.so"};
  for (int i = 0; i < 3 && !g_nccl.lib; i++)
    if (names[i] && names[i][0]) g_nccl.lib = dlopen(names[i], RTLD_NOW | RTLD_GLOBAL);
  if (!g_nccl.lib) { snprintf(t_nccl_err, sizeof t_nccl_err, "dlopen libnccl.so.2: %s", dlerror()); return B200_ERR_NCCL; }
#define NCCL_SYM(field, name)                                                             \
  *reinterpret_cast<void**>(&g_nccl.field) = dlsym(g_nccl.lib, name);                      \
  if (!g_nccl.field) { snprintf(t_nccl_err, sizeof t_nccl_err, "dlsym %s failed", name); return B200_ERR_NCCL; }
  NCCL_SYM(Broadcast, "ncclBroadcast")
  NCCL_SYM(GetErrorString, "ncclGetErrorString")
  NCCL_SYM(CommCount, "ncclCommCount")
  NCCL_SYM(CommUserRank, "ncclCommUserRank")
  NCCL_SYM(GetUniqueId, "ncclGetUniqueId")
  NCCL_SYM(CommInitRank, "ncclCommInitRank")
  NCCL_SYM(CommDestroy, "ncclCommDestroy")
#undef NCCL_SYM
  g_nccl.ok = true;
  return 0;
}
int nccl_check(ncclResult_t r, const char* what) {
  if (r == ncclSuccess) return 0;
  snprintf(t_nccl_err, sizeof t_nccl_err, "%s: %s", what, g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
  return B200_ERR_NCCL;
}

constexpr int kMaxSlices = 16;

}  // namespace

struct b200_rowpanel {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1, dev = -1;
  int m_max = 0, n = 0, k = 0, mode = 0;
  int nslices = 0;
  int trace = 0;            // diagnostics: timing events around every stage of the last call (b200_rowpanel_trace)
  cudaEvent_t tr[8 + 6 * kMaxSlices] = {};
  int reserve_sms = 0;      // SMs the GEMMs of all but the last K-slice leave to the exchange's copy kernels
  int k0[kMaxSlices + 1] = {};
  cudaStream_t comm_stream = nullptr;
  cudaEvent_t ev_start = nullptr, ev_b[kMaxSlices] = {}, ev_done = nullptr;
  // F16X2: planes of A_i (whole K) and of every slice of B, with their maxima; allocated once
  uint16_t* a_planes = nullptr; float* a_max = nullptr; long long a_pitch = 0;
  uint16_t* b_planes[kMaxSlices] = {}; float* b_max = nullptr; long long b_pitch = 0; int b_rows[kMaxSlices] = {};
  // host variant: device images + pipeline streams/events
  float *hA = nullptr, *hB = nullptr, *hC = nullptr;
  cudaStream_t h2d = nullptr, comp = nullptr, d2h = nullptr;
  cudaEvent_t ev_hb[kMaxSlices] = {}, ev_in[8] = {}, ev_out[8] = {};
  b200_packed_b* hpb = nullptr;
};

namespace {

void rowpanel_free(b200_rowpanel* rp) {
  if (!rp) return;
  if (rp->a_planes) cudaFree(rp->a_planes);
  if (rp->a_max) cudaFree(rp->a_max);
  for (int j = 0; j < kMaxSlices; j++) if (rp->b_planes[j]) cudaFree(rp->b_planes[j]);
  if (rp->b_max) cudaFree(rp->b_max);
  if (rp->hA) cudaFree(rp->hA);
  if (rp->hB) cudaFree(rp->hB);
  if (rp->hC) cudaFree(rp->hC);
  pack_destroy(rp->hpb);
  for (int j = 0; j < kMaxSlices; j++) { if (rp->ev_b[j]) cudaEventDestroy(rp->ev_b[j]); if (rp->ev_hb[j]) cudaEventDestroy(rp->ev_hb[j]); }
  for (auto& e : rp->tr) if (e) cudaEventDestroy(e);
  for (int j = 0; j < 8; j++) { if (rp->ev_in[j]) cudaEventDestroy(rp->ev_in[j]); if (rp->ev_out[j]) cudaEventDestroy(rp->ev_out[j]); }
  if (rp->ev_start) cudaEventDestroy(rp->ev_start);
  if (rp->ev_done) cudaEventDestroy(rp->ev_done);
  if (rp->comm_stream) cudaStreamDestroy(rp->comm_stream);
  if (rp->h2d) cudaStreamDestroy(rp->h2d);
  if (rp->comp) cudaStreamDestroy(rp->comp);
  if (rp->d2h) cudaStreamDestroy(rp->d2h);
  cudaGetLastError();
  delete rp;
}

// trace slots: 0 start(st) 1 after A split(st); per slice j: 8+6j+{0: bcast begin(comm), 1: bcast end(comm), 2: slice visible(st),
// 3: after split of the slice(st), 4: after its GEMM(st)}
inline void rp_mark(b200_rowpanel* rp, int slot, cudaStream_t s) {
  if (!rp->trace) return;
  if (!rp->tr[slot]) cudaEventCreate(&rp->tr[slot]);
  cudaEventRecord(rp->tr[slot], s);
}

#define RP_CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { cudaGetLastError(); return (int)e_; } } while (0)

// Enqueues the broadcast of B's K-slices on the comm stream (in place: root sends from, the others
// receive into, the operand buffer itself) and records one event per slice.
int rowpanel_broadcast(b200_rowpanel* rp, float* dB, int ldb, int n, int root, const cudaEvent_t* wait_per_slice) {
  for (int j = 0; j < rp->nslices; j++) {
    if (wait_per_slice && rp->rank == root) RP_CK(cudaStreamWaitEvent(rp->comm_stream, wait_per_slice[j], 0));
    if (rp->world > 1) {
      float* blk = dB + (size_t)rp->k0[j] * ldb;
      rp_mark(rp, 8 + 6 * j, rp->comm_stream);
      const size_t count = (size_t)(rp->k0[j + 1] - rp->k0[j]) * ldb - (size_t)(ldb - n);
      if (int rc = nccl_check(g_nccl.Broadcast(blk, blk, count, ncclFloat32, root, rp->comm, rp->comm_stream), "ncclBroadcast")) return rc;
    }
    rp_mark(rp, 8 + 6 * j + 1, rp->comm_stream);
    RP_CK(cudaEventRecord(rp->ev_b[j], rp->comm_stream));
  }
  return 0;
}

}  // namespace

extern "C" {

const char* b200_nccl_last_error(void) { return t_nccl_err; }
int b200_nccl_load(const char* path) { return nccl_load(path); }

int b200_comm_unique_id(void* id128) {
  if (!id128) return B200_ERR_BAD_ARG;
  if (int rc = nccl_load(nullptr)) return rc;
  return nccl_check(g_nccl.GetUniqueId(reinterpret_cast<ncclUniqueId*>(id128)), "ncclGetUniqueId");
}
int b200_comm_init_rank(void** comm_out, const void* id128, int rank, int world) {
  if (!comm_out || !id128 || world < 1 || rank < 0 || rank >= world) return B200_ERR_BAD_ARG;
  if (int rc = nccl_load(nullptr)) return rc;
  ncclUniqueId id;
  memcpy(&id, id128, sizeof id);
  ncclComm_t c = nullptr;
  if (int rc = nccl_check(g_nccl.CommInitRank(&c, world, id, rank), "ncclCommInitRank")) return rc;
  *comm_out = c;
  return 0;
}
int b200_comm_destroy(void* comm) {
  if (!comm) return 0;
  if (int rc = nccl_load(nullptr)) return rc;
  return nccl_check(g_nccl.CommDestroy(reinterpret_cast<ncclComm_t>(comm)), "ncclCommDestroy");
}

int b200_rowpanel_create(b200_rowpanel** out, void* nccl_comm, int m_local_max, int n, int k, int precision_mode,
                         const int* slice_rows, int n_slices) {
  if (!out) return B200_ERR_BAD_ARG;
  *out = nullptr;
  if (m_local_max <= 0 || n <= 0 || k <= 0 || n_slices < 0 || n_slices > kMaxSlices) return B200_ERR_BAD_ARG;
  int rc = ensure_device();
  if (rc) return rc;
  b200_rowpanel* rp = new b200_rowpanel();
  rp->dev = t_ctx->dev;
  rp->comm = reinterpret_cast<ncclComm_t>(nccl_comm);
  if (nccl_comm) {
    if ((rc = nccl_load(nullptr))) { delete rp; return rc; }
    if ((rc = nccl_check(g_nccl.CommCount(rp->comm, &rp->world), "ncclCommCount")) ||
        (rc = nccl_check(g_nccl.CommUserRank(rp->comm, &rp->rank), "ncclCommUserRank"))) { delete rp; return rc; }
  }
  rp->m_max = m_local_max; rp->n = n; rp->k = k;
  rp->mode = resolve_f32_mode(precision_mode);
  // K-slices: the caller's row counts (must add up to k, boundaries multiples of 8), else by default
  // one slice on a single rank, two slices weighted 1 : 3 up to 256 MB of B, equal ~256 MB slices beyond.
  if (n_slices > 0 && slice_rows) {
    int acc = 0;
    for (int j = 0; j < n_slices; j++) {
      if (slice_rows[j] <= 0 || (acc & 7)) { delete rp; return B200_ERR_BAD_ARG; }
      rp->k0[j] = acc; acc += slice_rows[j];
    }
    if (acc != k) { delete rp; return B200_ERR_BAD_ARG; }
    rp->k0[n_slices] = k; rp->nslices = n_slices;
  } else if (rp->world == 1 || k < 1024) {
    rp->nslices = 1; rp->k0[0] = 0; rp->k0[1] = k;
  } else {
    // Up to 256 MB of B: two slices, 1 : 3.  Every extra slice costs a GEMM launch with its own pass over C and
    // every ncclBroadcast a fixed latency, so small operands use few slices.  Larger operands (BASELINE config 5:
    // 1 GiB) amortise those costs: equal slices of ~256 MB, so that only a quarter of the exchange stays exposed.
    const double bytes = (double)k * n * 4.0;
    int ns = (int)((bytes + 268435455.0) / 268435456.0);
    ns = ns < 2 ? 2 : (ns > 8 ? 8 : ns);
    rp->nslices = ns;
    rp->k0[0] = 0;
    if (ns == 2) rp->k0[1] = (int)(((long long)k / 4 + 63) / 64 * 64);
    else for (int j = 1; j < ns; j++) rp->k0[j] = (int)(((long long)k * j / ns + 63) / 64 * 64);
    rp->k0[ns] = k;
  }
#define RP_TRY(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { cudaGetLastError(); rowpanel_free(rp); return (int)e_; } } while (0)
  RP_TRY(cudaStreamCreateWithFlags(&rp->comm_stream, cudaStreamNonBlocking));
  RP_TRY(cudaEventCreateWithFlags(&rp->ev_start, cudaEventDisableTiming));
  RP_TRY(cudaEventCreateWithFlags(&rp->ev_done, cudaEventDisableTiming));
  for (int j = 0; j < rp->nslices; j++) RP_TRY(cudaEventCreateWithFlags(&rp->ev_b[j], cudaEventDisableTiming));
  if (rp->mode == B200_F32_F16X2) {
    rp->a_pitch = plane_pitch(k);
    rp->b_pitch = plane_pitch(n);
    RP_TRY(cudaMalloc(&rp->a_planes, (size_t)2 * m_local_max * rp->a_pitch * 2));
    RP_TRY(cudaMalloc(&rp->a_max, (size_t)m_local_max * 4));
    RP_TRY(cudaMalloc(&rp->b_max, (size_t)rp->nslices * n * 4));
    for (int j = 0; j < rp->nslices; j++) {
      rp->b_rows[j] = b_plane_rows(rp->k0[j + 1] - rp->k0[j]);
      RP_TRY(cudaMalloc(&rp->b_planes[j], (size_t)2 * rp->b_rows[j] * rp->b_pitch * 2));
    }
  }
#undef RP_TRY
  *out = rp;
  return 0;
}

void b200_rowpanel_destroy(b200_rowpanel* rp) { rowpanel_free(rp); }
// Diagnostics: enable, run one call, then dump: out[0] = A split done, then per slice {bcast begin, bcast end, slice
// visible on the compute stream, split done, GEMM done}, all in ms after the call's first stream operation.
void b200_rowpanel_trace(b200_rowpanel* rp, int enable) { if (rp) rp->trace = enable; }
int b200_rowpanel_trace_dump(b200_rowpanel* rp, float* out, int cap) {
  if (!rp || !rp->trace || !rp->tr[0]) return 0;
  cudaDeviceSynchronize();
  int n = 0;
  auto get = [&](int slot) { float ms = -1.f; if (rp->tr[slot]) cudaEventElapsedTime(&ms, rp->tr[0], rp->tr[slot]); cudaGetLastError(); return ms; };
  if (n < cap) out[n++] = get(1);
  for (int j = 0; j < rp->nslices; j++)
    for (int e = 0; e < 5; e++) if (n < cap) out[n++] = get(8 + 6 * j + e);
  return n;
}
int b200_rowpanel_set_reserve_sms(b200_rowpanel* rp, int sms) {
  if (!rp || sms < -1 || sms > 64) return B200_ERR_BAD_ARG;
  if (sms == -1) return 0;
  rp->reserve_sms = sms;
  return 0;
}
int b200_rowpanel_slices(const b200_rowpanel* rp, int* bounds, int cap) {
  if (!rp) return 0;
  for (int j = 0; j <= rp->nslices && j < cap; j++) bounds[j] = rp->k0[j];
  return rp->nslices;
}

// One sharded product: C_local = A_local * B, B valid on `root` on entry and on every rank on return.
int b200_gemm_f32_rowpanel(b200_rowpanel* rp, int m_local, int n, int k, const float* dA, int lda, float* dB,
                           int ldb, float* dC, int ldc, int root, void* stream) {
  if (!rp || n != rp->n || k != rp->k || m_local > rp->m_max || root < 0 || root >= rp->world) return B200_ERR_BAD_ARG;
  int rc = check_args(m_local, n, k, dA, lda, dB, ldb, dC, ldc);
  if (rc < 0) return rc;
  if (!dB || ldb < n) return B200_ERR_BAD_ARG;            // B takes part in the exchange even when m_local == 0
  rc = ensure_device();
  if (rc) return rc;
  if (t_ctx->dev != rp->dev) return B200_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  // the exchange: comm stream starts once everything already queued on `st` (producer of B on the root,
  // earlier readers of the receive buffer elsewhere) is done
  rp_mark(rp, 0, st);
  RP_CK(cudaEventRecord(rp->ev_start, st));
  RP_CK(cudaStreamWaitEvent(rp->comm_stream, rp->ev_start, 0));
  if ((rc = rowpanel_broadcast(rp, dB, ldb, n, root, nullptr))) return rc;
  if (m_local == 0) {                                      // nothing to multiply: still order `st` after the exchange
    RP_CK(cudaStreamWaitEvent(st, rp->ev_b[rp->nslices - 1], 0));
    return 0;
  }
  if (rp->mode == B200_F32_F16X2) {
    // A_i -> fp16 planes while slice 0 of B travels
    if ((rc = launch_f16_split_rows(dA, lda, m_local, k, rp->a_max, rp->a_planes, rp->a_pitch, m_local, st))) return rc;
    RP_CK(cudaMemsetAsync(rp->b_max, 0, (size_t)rp->nslices * n * 4, st));
    rp_mark(rp, 1, st);
    for (int j = 0; j < rp->nslices; j++) {
      const int kk0 = rp->k0[j], kr = rp->k0[j + 1] - kk0;
      RP_CK(cudaStreamWaitEvent(st, rp->ev_b[j], 0));
      rp_mark(rp, 8 + 6 * j + 2, st);
      float* cmax = rp->b_max + (size_t)j * n;
      if ((rc = launch_f16_split_cols(dB + (size_t)kk0 * ldb, ldb, kr, n, cmax, rp->b_planes[j], rp->b_pitch,
                                      rp->b_rows[j], nullptr, 0, st))) return rc;
      rp_mark(rp, 8 + 6 * j + 3, st);
      const F16Operand oa{rp->a_planes + kk0, rp->a_pitch, m_local, rp->a_max};
      const F16Operand ob{rp->b_planes[j], rp->b_pitch, rp->b_rows[j], cmax};
      Call c{st};
      c.acc = j > 0;
      c.sm_reserve = rp->world > 1 && j + 1 < rp->nslices ? rp->reserve_sms : 0;   // a later slice is still being broadcast
      if ((rc = gemm_f16x2_core(B200_OP_N, B200_OP_N, m_local, n, kr, oa, ob, dC, ldc, c))) return rc;
      rp_mark(rp, 8 + 6 * j + 4, st);
    }
    return 0;
  }
  for (int j = 0; j < rp->nslices; j++) {
    const int kk0 = rp->k0[j], kr = rp->k0[j + 1] - kk0;
    RP_CK(cudaStreamWaitEvent(st, rp->ev_b[j], 0));
    const int reserve = rp->world > 1 && j + 1 < rp->nslices ? rp->reserve_sms : 0;
    if ((rc = gemm_f32(B200_OP_N, B200_OP_N, m_local, n, kr, 1.f, dA + kk0, lda, dB + (size_t)kk0 * ldb, ldb, j > 0 ? 1.f : 0.f,
                       dC, ldc, rp->mode, st, reserve))) return rc;
  }
  return 0;
}

// The same product with HOST operands and the CPU harnesses' contract C_local += A_local * B
// (aarch64/MMult0.cpp:16): B (host, root only) goes H2D in K-slices, each broadcast as soon as it has landed;
// every rank stages A_local / C_local in row blocks so the D2H of block i overlaps the H2D of block i + 1.
// Synchronous: returns when C_local is back in host memory.
int b200_gemm_f32_rowpanel_host(b200_rowpanel* rp, int m_local, int n, int k, const float* A, int lda, const float* B,
                                int ldb, float* C, int ldc, int root) {
  if (!rp || n != rp->n || k != rp->k || m_local > rp->m_max || m_local < 0 || root < 0 || root >= rp->world) return B200_ERR_BAD_ARG;
  if (m_local > 0 && (!A || !C || lda < k || ldc < n)) return B200_ERR_BAD_ARG;
  if (rp->rank == root && (!B || ldb < n)) return B200_ERR_BAD_ARG;
  int rc = ensure_device();
  if (rc) return rc;
  if (t_ctx->dev != rp->dev) return B200_ERR_BAD_ARG;
  if (!rp->h2d) {
    RP_CK(cudaStreamCreateWithFlags(&rp->h2d, cudaStreamNonBlocking));
    RP_CK(cudaStreamCreateWithFlags(&rp->comp, cudaStreamNonBlocking));
    RP_CK(cudaStreamCreateWithFlags(&rp->d2h, cudaStreamNonBlocking));
    for (int j = 0; j < rp->nslices; j++) RP_CK(cudaEventCreateWithFlags(&rp->ev_hb[j], cudaEventDisableTiming));
    for (int j = 0; j < 8; j++) {
      RP_CK(cudaEventCreateWithFlags(&rp->ev_in[j], cudaEventDisableTiming));
      RP_CK(cudaEventCreateWithFlags(&rp->ev_out[j], cudaEventDisableTiming));
    }
    RP_CK(cudaMalloc(&rp->hA, (size_t)rp->m_max * k * 4));
    RP_CK(cudaMalloc(&rp->hB, (size_t)k * n * 4));
    RP_CK(cudaMalloc(&rp->hC, (size_t)rp->m_max * n * 4));
  }
  // B: root uploads slice by slice; the broadcast of slice j waits for its upload only
  if (rp->rank == root)
    for (int j = 0; j < rp->nslices; j++) {
      const int kk0 = rp->k0[j], kr = rp->k0[j + 1] - kk0;
      RP_CK(cudaMemcpy2DAsync(rp->hB + (size_t)kk0 * n, (size_t)n * 4, B + (size_t)kk0 * ldb, (size_t)ldb * 4, (size_t)n * 4, kr,
                              cudaMemcpyHostToDevice, rp->h2d));
      RP_CK(cudaEventRecord(rp->ev_hb[j], rp->h2d));
    }
  if ((rc = rowpanel_broadcast(rp, rp->hB, n, n, root, rp->ev_hb))) return rc;
  // A_i / C_i in row blocks (whole pair tiles); every block multiplies the complete B
  const int blocks = m_local >= 2048 ? 4 : 1;
  const int rows_per = blocks == 1 ? (m_local > 0 ? m_local : 1) : (((m_local + blocks - 1) / blocks + 255) & ~255);
  RP_CK(cudaStreamWaitEvent(rp->comp, rp->ev_b[rp->nslices - 1], 0));
  int nb = 0;
  for (int r0 = 0; r0 < m_local; r0 += rows_per, nb++) {
    const int rows = m_local - r0 < rows_per ? m_local - r0 : rows_per;
    float* dAi = rp->hA + (size_t)r0 * k;
    float* dCi = rp->hC + (size_t)r0 * n;
    RP_CK(cudaMemcpy2DAsync(dAi, (size_t)k * 4, A + (size_t)r0 * lda, (size_t)lda * 4, (size_t)k * 4, rows, cudaMemcpyHostToDevice, rp->h2d));
    RP_CK(cudaMemcpy2DAsync(dCi, (size_t)n * 4, C + (size_t)r0 * ldc, (size_t)ldc * 4, (size_t)n * 4, rows, cudaMemcpyHostToDevice, rp->h2d));
    RP_CK(cudaEventRecord(rp->ev_in[nb], rp->h2d));
    RP_CK(cudaStreamWaitEvent(rp->comp, rp->ev_in[nb], 0));
    if ((rc = gemm_f32(B200_OP_N, B200_OP_N, rows, n, k, 1.f, dAi, k, rp->hB, n, 1.f, dCi, n, rp->mode, rp->comp))) return rc;
    RP_CK(cudaEventRecord(rp->ev_out[nb], rp->comp));
    RP_CK(cudaStreamWaitEvent(rp->d2h, rp->ev_out[nb], 0));
    RP_CK(cudaMemcpy2DAsync(C + (size_t)r0 * ldc, (size_t)ldc * 4, dCi, (size_t)n * 4, (size_t)n * 4, rows, cudaMemcpyDeviceToHost, rp->d2h));
  }
  RP_CK(cudaStreamSynchronize(rp->d2h));
  RP_CK(cudaStreamSynchronize(rp->comp));
  RP_CK(cudaStreamSynchronize(rp->comm_stream));
  return 0;
}

}  // extern "C"
