// rowpanel_demo.cpp — a C++ host for the multi-GPU entry points of include/b200gemm.h (no Python, no torch).
//
// north_star: "host code stays C++ calling the kernel through a thin C-ABI ... Large square problems shard C by
// row-panels across the box's GPUs with one NCCL broadcast of B over NVLink".  One process, one host thread per GPU
// (the library's state is per device): rank 0 creates the NCCL id (b200_comm_unique_id), every thread joins
// (b200_comm_init_rank), builds a plan (b200_rowpanel_create) and runs the sharded product
// (b200_gemm_f32_rowpanel): rank i owns a row panel of A and C, B lives on rank 0 and is broadcast inside every call.
// Inputs follow the reference's generator (cuda/random_matrix.cpp:6-16: 2*drand48()-1), timing follows its harness
// (cuda/test_MMult.cpp:98-118: NREPEATS back-to-back calls between two events, operands resident), the check follows
// its oracle (REF_MMult: here a double-precision dot product on sampled rows, max |diff| / max |ref|).
//
//   rowpanel_demo.x [gpus=all] [m_per_gpu=4096] [n=4096] [k=4096] [repeats=20]
//
// Output: one Octave-style row per run, "gpus  GFLOP/s(total)  max_rel_err", in the spirit of the reference's output_*.m.
#include <cuda_runtime.h>

#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "../../include/b200gemm.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { std::fprintf(stderr, "CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); std::exit(2); } } while (0)
#define BK(x) do { int rc_ = (x); if (rc_ != 0) { std::fprintf(stderr, "b200gemm error %d (%s) %s at %s:%d\n", rc_, b200_gemm_strerror(rc_), b200_nccl_last_error(), __FILE__, __LINE__); std::exit(3); } } while (0)

struct Shared {
  int world, m, n, k, repeats;
  unsigned char id[128];
  std::vector<float> a, b;            // A (world*m x k), B (k x n), host copies for the check
  std::vector<double> ms;             // per rank
  std::vector<double> err;            // per rank
  std::atomic<int> ready{0};
};

static void worker(Shared* s, int rank) {
  CK(cudaSetDevice(rank));
  void* comm = nullptr;
  if (s->world > 1) BK(b200_comm_init_rank(&comm, s->id, rank, s->world));
  const size_t mk = (size_t)s->m * s->k, kn = (size_t)s->k * s->n, mn = (size_t)s->m * s->n;
  float *dA, *dB, *dC;
  CK(cudaMalloc(&dA, mk * 4));
  CK(cudaMalloc(&dB, kn * 4));
  CK(cudaMalloc(&dC, mn * 4));
  CK(cudaMemcpy(dA, s->a.data() + (size_t)rank * mk, mk * 4, cudaMemcpyHostToDevice));
  if (rank == 0) CK(cudaMemcpy(dB, s->b.data(), kn * 4, cudaMemcpyHostToDevice));
  else CK(cudaMemset(dB, 0xff, kn * 4));                                  // NaNs: the exchange must overwrite them
  b200_rowpanel* plan = nullptr;
  BK(b200_rowpanel_create(&plan, comm, s->m, s->n, s->k, B200_F32_AUTO, nullptr, 0));
  cudaStream_t st;
  CK(cudaStreamCreate(&st));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  for (int i = 0; i < 3; i++) BK(b200_gemm_f32_rowpanel(plan, s->m, s->n, s->k, dA, s->k, dB, s->n, dC, s->n, 0, st));
  CK(cudaStreamSynchronize(st));
  s->ready.fetch_add(1);
  while (s->ready.load() < s->world) std::this_thread::yield();           // all ranks start the timed loop together
  CK(cudaEventRecord(e0, st));
  for (int i = 0; i < s->repeats; i++) BK(b200_gemm_f32_rowpanel(plan, s->m, s->n, s->k, dA, s->k, dB, s->n, dC, s->n, 0, st));
  CK(cudaEventRecord(e1, st));
  CK(cudaEventSynchronize(e1));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  s->ms[rank] = ms / s->repeats;
  // check 8 rows of this rank's panel against a double-precision dot product of the host operands
  std::vector<float> c(mn);
  CK(cudaMemcpy(c.data(), dC, mn * 4, cudaMemcpyDeviceToHost));
  double max_err = 0.0, max_ref = 0.0;
  for (int t = 0; t < 8; t++) {
    const int i = (int)(((long long)t * (s->m - 1)) / 7);
    const float* ai = s->a.data() + ((size_t)rank * s->m + i) * s->k;
    for (int j = 0; j < s->n; j += 7) {
      double ref = 0.0;
      for (int p = 0; p < s->k; p++) ref += (double)ai[p] * (double)s->b[(size_t)p * s->n + j];
      max_err = std::fmax(max_err, std::fabs(ref - (double)c[(size_t)i * s->n + j]));
      max_ref = std::fmax(max_ref, std::fabs(ref));
    }
  }
  s->err[rank] = max_err / (max_ref > 0 ? max_ref : 1.0);
  b200_rowpanel_destroy(plan);
  if (comm) b200_comm_destroy(comm);
  cudaFree(dA); cudaFree(dB); cudaFree(dC);
}

int main(int argc, char** argv) {
  int ndev = 0;
  CK(cudaGetDeviceCount(&ndev));
  Shared s;
  s.world = argc > 1 ? std::atoi(argv[1]) : ndev;
  s.m = argc > 2 ? std::atoi(argv[2]) : 4096;
  s.n = argc > 3 ? std::atoi(argv[3]) : 4096;
  s.k = argc > 4 ? std::atoi(argv[4]) : 4096;
  s.repeats = argc > 5 ? std::atoi(argv[5]) : 20;
  if (s.world < 1 || s.world > ndev) { std::fprintf(stderr, "%d GPUs requested, %d present\n", s.world, ndev); return 1; }
  if (b200_gemm_device_ok() != 0) { std::fprintf(stderr, "no usable sm_90 device (there is no CPU fallback)\n"); return 1; }
  if (s.world > 1) BK(b200_comm_unique_id(s.id));
  srand48(20260923);
  s.a.resize((size_t)s.world * s.m * s.k);
  s.b.resize((size_t)s.k * s.n);
  for (auto& v : s.a) v = 2.0f * (float)drand48() - 1.0f;                 // cuda/random_matrix.cpp:12
  for (auto& v : s.b) v = 2.0f * (float)drand48() - 1.0f;
  s.ms.assign(s.world, 0.0);
  s.err.assign(s.world, 0.0);
  std::vector<std::thread> th;
  for (int r = 0; r < s.world; r++) th.emplace_back(worker, &s, r);
  for (auto& t : th) t.join();
  double ms = 0.0, err = 0.0;
  for (int r = 0; r < s.world; r++) { ms = std::fmax(ms, s.ms[r]); err = std::fmax(err, s.err[r]); }
  const double gflops = 2.0 * s.world * s.m * (double)s.n * s.k / (ms * 1e-3) / 1e9;
  std::printf("version = 'b200gemm_rowpanel_cxx';\n%% %s; M = %d x %d rows, N = %d, K = %d, B broadcast from rank 0 inside every call\n",
              b200_gemm_version(), s.world, s.m, s.n, s.k);
  std::printf("MY_MMult = [\n%d %.2f %le \n];\n", s.world, gflops, err);
  return err <= 1e-5 ? 0 : 4;
}
