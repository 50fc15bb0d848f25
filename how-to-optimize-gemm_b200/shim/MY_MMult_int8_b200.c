/* MY_MMult_int8_b200.c — plug-in for the reference's int8 harness (C linkage):
 *   void MY_MMult(int m, int n, int k, int8_t* a, int lda, int8_t* b, int ldb, int32_t* c, int ldc,
 *                 double* packZ_cost, double* packN_cost, double* kernel_cost)
 *   aarch64-int8/test_MMult.c:9,98; reference definition aarch64-int8/MMult_4x8_21.c:81-86.
 * C = A*B, int8 x int8 -> int32, any m,n,k; the three cost out-params are zeroed exactly as the
 * reference does (MMult_4x8_21.c:88) — there is no packZ/packN pass here (TMA stages A; the library transposes B once per call for the tensor core). */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/b200gemm.h"

void MY_MMult(int m, int n, int k, int8_t* a, int lda, int8_t* b, int ldb, int32_t* c, int ldc,
              double* packZ_cost, double* packN_cost, double* kernel_cost) {
  *packN_cost = *packZ_cost = *kernel_cost = 0.0;
  int rc = b200_gemm_s8s32_host(m, n, k, a, lda, b, ldb, c, ldc);
  if (rc != 0) {
    fprintf(stderr, "b200gemm error in MY_MMult(int8): code=%d \"%s\"\n", rc, b200_gemm_strerror(rc));
    exit(EXIT_FAILURE);
  }
}
