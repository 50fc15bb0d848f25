// test_MMult_b200.cpp — sweep driver for libb200gemm, the GPU counterpart of the reference's
// benchmark/verify harness (cuda/test_MMult.cpp:21-146).  Same protocol, same output:
//
//   version = '<name>';                                   (cuda/makefile:43)
//   GPU Device 0: "<name>" with compute capability x.y   (cuda/test_MMult.cpp:32-33)
//
//   MY_MMult = [
//   <N> <GFLOP/s> <max|diff|>                             (cuda/test_MMult.cpp:128, "%d %.2f %le \n")
//   ];
//
// so cuda/plot.py:5-28 parses the files unchanged.  Differences, all deliberate (SURVEY App. B):
// inputs are seeded (srand48) per size, W warm-up launches precede the timed NREPEATS launches
// (the reference times the cold first launch, B-3), and dtype/mode are selectable.
//
// The third column here is a SELF-CHECK against this library's strict CUDA-core kernels (the
// sequential-k FFMA / integer path), not the oracle: product code never links oracle/.  Parity
// against REF_MMult proper is the job of tests/ and of the reference's own test_MMult.cpp linked
// against shim/MY_MMult_b200.cpp (see INTEGRATION.md).
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/b200gemm.h"

#define CUDA_OK(x)                                                                      \
  do {                                                                                  \
    cudaError_t e_ = (x);                                                               \
    if (e_ != cudaSuccess) {                                                            \
      std::fprintf(stderr, "CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      std::exit(EXIT_FAILURE);                                                          \
    }                                                                                   \
  } while (0)
#define GEMM_OK(x)                                                                      \
  do {                                                                                  \
    int r_ = (x);                                                                       \
    if (r_ != 0) {                                                                      \
      std::fprintf(stderr, "b200gemm error %d (%s) at %s:%d\n", r_, b200_gemm_strerror(r_), __FILE__, __LINE__); \
      std::exit(EXIT_FAILURE);                                                          \
    }                                                                                   \
  } while (0)

static uint16_t bf16_rne(float x) {
  uint32_t u;
  std::memcpy(&u, &x, 4);
  u += 0x7FFFu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
static float bf16_up(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float x;
  std::memcpy(&x, &u, 4);
  return x;
}

struct Opts {
  std::string dtype = "f32", mode = "auto", version = "b200gemm";
  int first = 256, last = 4096, inc = 256, reps = 20, warmup = 3, check = 1;
  int M = -1, N = -1, K = -1;
  long seed = 1;
};

static int mode_of(const std::string& s) {
  if (s == "strict") return B200_F32_STRICT;
  if (s == "tf32") return B200_F32_TF32;
  if (s == "bf16x3") return B200_F32_BF16X3;
  if (s == "bf16x2") return B200_F32_BF16X2;
  return B200_F32_AUTO;
}

int main(int argc, char** argv) {
  Opts o;
  for (int i = 1; i < argc; i++) {
    std::string a = argv[i];
    auto next = [&]() -> const char* { return i + 1 < argc ? argv[++i] : ""; };
    if (a == "--dtype") o.dtype = next();
    else if (a == "--mode") o.mode = next();
    else if (a == "--version") o.version = next();
    else if (a == "--first") o.first = std::atoi(next());
    else if (a == "--last") o.last = std::atoi(next());
    else if (a == "--inc") o.inc = std::atoi(next());
    else if (a == "--reps") o.reps = std::atoi(next());
    else if (a == "--warmup") o.warmup = std::atoi(next());
    else if (a == "--seed") o.seed = std::atol(next());
    else if (a == "--check") o.check = std::atoi(next());
    else if (a == "--m") o.M = std::atoi(next());
    else if (a == "--n") o.N = std::atoi(next());
    else if (a == "--k") o.K = std::atoi(next());
    else { std::fprintf(stderr, "unknown option %s\n", a.c_str()); return 2; }
  }
  cudaDeviceProp prop;
  CUDA_OK(cudaSetDevice(0));
  CUDA_OK(cudaGetDeviceProperties(&prop, 0));
  GEMM_OK(b200_gemm_device_ok());
  std::printf("version = '%s';\n", o.version.c_str());
  std::printf("GPU Device %d: \"%s\" with compute capability %d.%d\n\n", 0, prop.name, prop.major, prop.minor);
  std::printf("MY_MMult = [\n");
  cudaEvent_t t0, t1;
  CUDA_OK(cudaEventCreate(&t0));
  CUDA_OK(cudaEventCreate(&t1));
  const int mode = mode_of(o.mode);
  const bool is_bf16 = o.dtype == "bf16", is_s8 = o.dtype == "s8";
  const size_t esz = is_bf16 ? 2 : is_s8 ? 1 : 4;

  for (int p = o.first; p <= o.last; p += o.inc) {
    const int m = o.M == -1 ? p : o.M, n = o.N == -1 ? p : o.N, k = o.K == -1 ? p : o.K;
    const int lda = k, ldb = n, ldc = n;      // cuda/test_MMult.cpp:62
    const size_t na = (size_t)m * k, nb = (size_t)k * n, nc = (size_t)m * n;
    // inputs: uniform(-1,1) from drand48 (cuda/random_matrix.cpp:12), seeded per size; int8: [-127,127]
    std::vector<float> a(na), b(nb);
    srand48(o.seed + p);
    for (size_t i = 0; i < na; i++) a[i] = (float)(2.0 * (double)(float)drand48() - 1.0);
    for (size_t i = 0; i < nb; i++) b[i] = (float)(2.0 * (double)(float)drand48() - 1.0);
    void *dA, *dB, *dC;
    float *fA = nullptr, *fB = nullptr, *fC = nullptr;   // fp32 images for the strict cross-check
    CUDA_OK(cudaMalloc(&dA, na * esz));
    CUDA_OK(cudaMalloc(&dB, nb * esz));
    CUDA_OK(cudaMalloc(&dC, nc * 4));
    std::vector<int8_t> a8, b8;
    if (is_bf16) {
      std::vector<uint16_t> ha(na), hb(nb);
      for (size_t i = 0; i < na; i++) { ha[i] = bf16_rne(a[i]); a[i] = bf16_up(ha[i]); }
      for (size_t i = 0; i < nb; i++) { hb[i] = bf16_rne(b[i]); b[i] = bf16_up(hb[i]); }
      CUDA_OK(cudaMemcpy(dA, ha.data(), na * 2, cudaMemcpyHostToDevice));
      CUDA_OK(cudaMemcpy(dB, hb.data(), nb * 2, cudaMemcpyHostToDevice));
    } else if (is_s8) {
      a8.resize(na); b8.resize(nb);
      for (size_t i = 0; i < na; i++) a8[i] = (int8_t)lrintf(a[i] * 127.0f);
      for (size_t i = 0; i < nb; i++) b8[i] = (int8_t)lrintf(b[i] * 127.0f);
      CUDA_OK(cudaMemcpy(dA, a8.data(), na, cudaMemcpyHostToDevice));
      CUDA_OK(cudaMemcpy(dB, b8.data(), nb, cudaMemcpyHostToDevice));
    } else {
      CUDA_OK(cudaMemcpy(dA, a.data(), na * 4, cudaMemcpyHostToDevice));
      CUDA_OK(cudaMemcpy(dB, b.data(), nb * 4, cudaMemcpyHostToDevice));
    }
    auto run = [&]() {
      if (is_bf16) GEMM_OK(b200_gemm_bf16(m, n, k, (const uint16_t*)dA, lda, (const uint16_t*)dB, ldb, dC, ldc, B200_OUT_F32, nullptr));
      else if (is_s8) GEMM_OK(b200_gemm_s8s32(m, n, k, (const int8_t*)dA, lda, (const int8_t*)dB, ldb, (int32_t*)dC, ldc, nullptr));
      else GEMM_OK(b200_gemm_f32(m, n, k, (const float*)dA, lda, (const float*)dB, ldb, (float*)dC, ldc, mode, nullptr));
    };
    for (int w = 0; w < o.warmup; w++) run();
    CUDA_OK(cudaEventRecord(t0, nullptr));
    for (int r = 0; r < o.reps; r++) run();              // the hot loop of cuda/test_MMult.cpp:100-103
    CUDA_OK(cudaEventRecord(t1, nullptr));
    CUDA_OK(cudaEventSynchronize(t1));
    float ms = 0.f;
    CUDA_OK(cudaEventElapsedTime(&ms, t0, t1));
    const double gflops = 2.0 * m * n * k * 1e-9 / (ms / o.reps / 1000.0);

    double diff = NAN;
    if (o.check) {
      std::vector<float> got(nc), want(nc);
      CUDA_OK(cudaMemcpy(got.data(), dC, nc * 4, cudaMemcpyDeviceToHost));
      if (is_s8) {
        // cross-check through the host entry on a row subset (generic int8 CUDA-core path has the
        // same exact semantics; use unaligned ld to force it)
        const int rows = m < 64 ? m : 64;
        std::vector<int32_t> w32((size_t)rows * n);
        std::vector<int8_t> apad((size_t)rows * (k + 1)), bpad((size_t)k * (n + 1));
        for (int i = 0; i < rows; i++) std::memcpy(&apad[(size_t)i * (k + 1)], &a8[(size_t)i * k], k);
        for (int i = 0; i < k; i++) std::memcpy(&bpad[(size_t)i * (n + 1)], &b8[(size_t)i * n], n);
        int8_t *pA, *pB; int32_t* pC;
        CUDA_OK(cudaMalloc(&pA, apad.size())); CUDA_OK(cudaMalloc(&pB, bpad.size())); CUDA_OK(cudaMalloc(&pC, w32.size() * 4));
        CUDA_OK(cudaMemcpy(pA, apad.data(), apad.size(), cudaMemcpyHostToDevice));
        CUDA_OK(cudaMemcpy(pB, bpad.data(), bpad.size(), cudaMemcpyHostToDevice));
        GEMM_OK(b200_gemm_s8s32(rows, n, k, pA, k + 1, pB, n + 1, pC, n, nullptr));
        CUDA_OK(cudaMemcpy(w32.data(), pC, w32.size() * 4, cudaMemcpyDeviceToHost));
        cudaFree(pA); cudaFree(pB); cudaFree(pC);
        const int32_t* g32 = reinterpret_cast<const int32_t*>(got.data());
        long long mx = 0;
        for (size_t i = 0; i < w32.size(); i++) { long long d = llabs((long long)g32[i] - w32[i]); if (d > mx) mx = d; }
        diff = (double)mx;
      } else {
        CUDA_OK(cudaMalloc(&fC, nc * 4));
        if (is_bf16) {
          CUDA_OK(cudaMalloc(&fA, na * 4)); CUDA_OK(cudaMalloc(&fB, nb * 4));
          CUDA_OK(cudaMemcpy(fA, a.data(), na * 4, cudaMemcpyHostToDevice));
          CUDA_OK(cudaMemcpy(fB, b.data(), nb * 4, cudaMemcpyHostToDevice));
        }
        GEMM_OK(b200_gemm_f32(m, n, k, is_bf16 ? fA : (const float*)dA, lda, is_bf16 ? fB : (const float*)dB, ldb, fC, ldc, B200_F32_STRICT, nullptr));
        CUDA_OK(cudaMemcpy(want.data(), fC, nc * 4, cudaMemcpyDeviceToHost));
        double mx = 0;
        for (size_t i = 0; i < nc; i++) {
          double d = std::fabs((double)got[i] - (double)want[i]);
          if (!(d == d)) { mx = NAN; break; }
          if (d > mx) mx = d;
        }
        diff = mx;
        cudaFree(fA); cudaFree(fB); cudaFree(fC); fA = fB = fC = nullptr;
      }
      if (!(diff <= 0.5)) {                        // cuda/test_MMult.cpp:124-127
        std::printf("diff too big !\n");
        std::exit(-1);
      }
    }
    std::printf("%d %.2f %le \n", p, gflops, diff);
    std::fflush(stdout);
    cudaFree(dA); cudaFree(dB); cudaFree(dC);
  }
  std::printf("];\n");
  return 0;
}
