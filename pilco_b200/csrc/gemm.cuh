// gemm.cuh -- factorize.cu's batched fp64 GEMM (DMMA path), for the other translation units that reuse it:
//   C = alpha op(A) op(B) + beta C, row-major, op = transpose where ta / tb is set; batch z at A + z sa, B + z sb,
//   C + z sc; grid (ceil(n / 64), ceil(m / 64), batch), no split over k.  Fixed order: deterministic.
#pragma once
#include <cuda_runtime.h>

int gemm(cudaStream_t st, int batch, int m, int n, int k, int ta, int tb, double alpha,
         const double* A, int lda, long long sa, const double* B, int ldb, long long sb,
         double beta, double* C, int ldc, long long sc);
