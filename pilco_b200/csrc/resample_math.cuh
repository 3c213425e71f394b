// resample_math.cuh -- the Gaussian refit of the resampled particle rollout (DESIGN.md section 26): the column-by-column
// Cholesky factor of a sample covariance with its degenerate-column rule, and its reverse.  Plain scalar code on
// row-major n x n arrays (n <= PILCO_MAX_D), run by one thread of particles_resample.cu's kernels on shared memory and
// (for the CPU test of the formulas, tests/test_particles_resample_host.py) by a host compiler.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define PR_HD __host__ __device__ __forceinline__
#else
#define PR_HD inline
#endif

#define PR_TAU 1e-12            // a pivot d_j <= PR_TAU S_jj (or S_jj <= 0) makes column j degenerate

// L = chol(S) from S's lower triangle, column by column (left-looking); L's upper triangle is written 0.  Column j:
//   d_j = S_jj - sum_{k<j} L_jk^2;  degenerate (d_j <= PR_TAU S_jj, or S_jj <= 0, or NaN): the column is 0;
//   otherwise L_jj = sqrt(d_j), L_ij = (S_ij - sum_{k<j} L_ik L_jk) / L_jj for i > j.
// A degenerate column has L_jj = 0 exactly and every other L_jj > 0, which is how the reverse tells them apart.
PR_HD void pr_chol(const double* S, double* L, int n) {
    for (int j = 0; j < n; ++j) {
        const double sjj = S[j * n + j];
        double d = sjj;
        for (int k = 0; k < j; ++k) d = fma(-L[j * n + k], L[j * n + k], d);
        const bool ok = sjj > 0.0 && d > PR_TAU * sjj;
        const double piv = ok ? sqrt(d) : 0.0;
        for (int i = 0; i < j; ++i) L[i * n + j] = 0.0;
        L[j * n + j] = piv;
        for (int i = j + 1; i < n; ++i) {
            double s = S[i * n + j];
            for (int k = 0; k < j; ++k) s = fma(-L[i * n + k], L[j * n + k], s);
            L[i * n + j] = ok ? s / piv : 0.0;
        }
    }
}

// The reverse of pr_chol as executed: Sb (lower triangle; the upper is written 0) = d value / d S_ij (i >= j) from
// Lb = d value / d L (lower triangle, used as scratch and overwritten).  Columns j = n-1 .. 0; a degenerate column
// (L_jj = 0) is constant and contributes nothing.
PR_HD void pr_chol_bwd(const double* L, double* Lb, double* Sb, int n) {
    for (int i = 0; i < n * n; ++i) Sb[i] = 0.0;
    for (int j = n - 1; j >= 0; --j) {
        const double piv = L[j * n + j];
        if (!(piv > 0.0)) continue;
        double pb = Lb[j * n + j];
        for (int i = j + 1; i < n; ++i) {            // L_ij = n_ij / L_jj
            const double nb = Lb[i * n + j] / piv;
            pb = fma(-nb, L[i * n + j], pb);
            Sb[i * n + j] += nb;
            for (int k = 0; k < j; ++k) {
                Lb[i * n + k] = fma(-nb, L[j * n + k], Lb[i * n + k]);
                Lb[j * n + k] = fma(-nb, L[i * n + k], Lb[j * n + k]);
            }
        }
        const double db = pb / (2.0 * piv);          // L_jj = sqrt(d_j)
        Sb[j * n + j] += db;
        for (int k = 0; k < j; ++k) Lb[j * n + k] = fma(-2.0 * db, L[j * n + k], Lb[j * n + k]);
    }
}
