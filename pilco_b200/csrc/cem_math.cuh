// cem_math.cuh -- the cross-entropy method's per-element work (DESIGN.md section 31): the rank order, one step of the
// bitonic sort, the elite refit of one (t, u) element and the clipped draw.  Plain scalar code, usable from the device
// kernels of particles_cem.cu and (for the CPU test against the numpy oracle, tests/test_particles_cem_host.py) from a
// host compiler.  Products and sums go through cem_mul / cem_add, which the device compiler may not contract into an
// fma, so that a host build without contraction computes the device's bits.
#pragma once
#include <math.h>
#include <stddef.h>

#if defined(__CUDACC__)
#define CEM_HD __host__ __device__ __forceinline__
#else
#define CEM_HD inline
#endif

CEM_HD double cem_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

CEM_HD double cem_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}

// the rank order: (va, ia) comes before (vb, ib) when va is the larger value; a NaN comes after every number; ties (and
// two NaNs) go to the lower index.  A strict total order on distinct indices.
CEM_HD bool cem_before(double va, int ia, double vb, int ib) {
    const bool an = va != va, bn = vb != vb;
    if (an != bn) return bn;
    if (!an && va != vb) return va > vb;
    return ia < ib;
}

// one compare-exchange of the bitonic sort of N = 2^m (value, index) pairs into rank order: stage (k, j), element i.
// Within a stage the pairs (i, i ^ j) are disjoint, so the i of a stage may run in any order or in parallel.
CEM_HD void cem_bitonic_step(double* v, int* ix, int i, int j, int k) {
    const int l = i ^ j;
    if (l <= i) return;
    const bool up = (i & k) == 0;                       // this block sorts into rank order (else the reverse)
    const bool swap = up ? cem_before(v[l], ix[l], v[i], ix[i]) : cem_before(v[i], ix[i], v[l], ix[l]);
    if (swap) {
        const double tv = v[i]; v[i] = v[l]; v[l] = tv;
        const int ti = ix[i]; ix[i] = ix[l]; ix[l] = ti;
    }
}

// the refit of element e of the [H,U] sampling distribution from the ke elites (order[0 .. ke), rows of cand [K, HU]):
//   m_e = sum_q c_q / ke,  v_e = sum_q (c_q - m_e)^2 / ke  (rank order, two passes)
//   mean <- alpha mean + (1 - alpha) m_e,  std <- sqrt(alpha std^2 + (1 - alpha) v_e)
CEM_HD void cem_refit(const double* cand, const int* order, int ke, size_t HU, size_t e, double alpha, double* mean,
                      double* std) {
    double s = 0.0;
    for (int q = 0; q < ke; ++q) s = cem_add(s, cand[(size_t)order[q] * HU + e]);
    const double m = s / ke;
    double s2 = 0.0;
    for (int q = 0; q < ke; ++q) {
        const double d = cand[(size_t)order[q] * HU + e] - m;
        s2 = cem_add(s2, cem_mul(d, d));
    }
    const double v = s2 / ke, beta = 1.0 - alpha, sd = *std;
    *mean = cem_add(cem_mul(alpha, *mean), cem_mul(beta, m));
    *std = sqrt(cem_add(cem_mul(alpha, cem_mul(sd, sd)), cem_mul(beta, v)));
}

// clip(x, lo, hi); a NaN stays NaN
CEM_HD double cem_clip(double x, double lo, double hi) { return x < lo ? lo : (x > hi ? hi : x); }

// candidate row k's element at (mean, std): row 0 is clip(mean), row k >= 1 clip(mean + std xi)
CEM_HD double cem_draw(int k, double mean, double std, double xi, double lo, double hi) {
    return cem_clip(k == 0 ? mean : cem_add(mean, cem_mul(std, xi)), lo, hi);
}
