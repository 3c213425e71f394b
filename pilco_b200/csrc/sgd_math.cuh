// sgd_math.cuh -- the stochastic optimiser's per-element work (DESIGN.md section 32): Philox4x32-10 and the normals it
// gives, and the Adam step of one parameter with the fixed-order norm of a gradient row.  Plain scalar code, usable
// from the device kernels of particles_sgd.cu and (for the CPU test against the numpy oracle,
// tests/test_particles_sgd_host.py) from a host compiler.  Products, sums, quotients and square roots go through
// sgd_mul / sgd_add / sgd_div / sgd_sqrt, which the device compiler may not contract into an fma, so that a host build
// without contraction computes the device's bits.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define SGD_HD __host__ __device__ __forceinline__
#else
#define SGD_HD inline
#endif

#define SGD_LANES 256           // the lanes of the gradient norm's fixed summation order (and the Adam kernel's CTA)

SGD_HD double sgd_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

SGD_HD double sgd_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}

SGD_HD double sgd_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

SGD_HD double sgd_sqrt(double a) {
#if defined(__CUDA_ARCH__)
    return __dsqrt_rn(a);
#else
    return sqrt(a);
#endif
}

// ---- Philox4x32-10 (Salmon et al. 2011; curand's Philox4_32_10 with the counter set directly) ----------------------
SGD_HD void sgd_mulhilo(uint32_t a, uint32_t b, uint32_t* hi, uint32_t* lo) {
    const uint64_t p = (uint64_t)a * b;
    *hi = (uint32_t)(p >> 32);
    *lo = (uint32_t)p;
}

// the ten rounds on counter c[4] with key (k0, k1), in place
SGD_HD void sgd_philox(uint32_t c[4], uint32_t k0, uint32_t k1) {
    for (int r = 0; r < 10; ++r) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        uint32_t hi0, lo0, hi1, lo1;
        sgd_mulhilo(0xD2511F53u, c[0], &hi0, &lo0);
        sgd_mulhilo(0xCD9E8D57u, c[2], &hi1, &lo1);
        const uint32_t c1 = c[1], c3 = c[3];
        c[0] = hi1 ^ c1 ^ k0;
        c[1] = lo1;
        c[2] = hi0 ^ c3 ^ k1;
        c[3] = lo0;
    }
}

// the uniform in (0, 1) of two Philox words: (((a << 32 | b) >> 11) + 0.5) 2^-53, exact
SGD_HD double sgd_uniform(uint32_t a, uint32_t b) {
    const uint64_t x = ((uint64_t)a << 32 | b) >> 11;
    return ((double)x + 0.5) * 1.1102230246251565404e-16;
}

// the two uniforms (u1, u2) of pair j of (seed, stream, iteration): Philox of the counter (j low, j high, stream,
// iteration) under the key (seed low, seed high)
SGD_HD void sgd_pair_uniforms(uint64_t seed, uint32_t stream, uint32_t iteration, uint64_t j, double* u1,
                              double* u2) {
    uint32_t c[4] = {(uint32_t)j, (uint32_t)(j >> 32), stream, iteration};
    sgd_philox(c, (uint32_t)seed, (uint32_t)(seed >> 32));
    *u1 = sgd_uniform(c[0], c[1]);
    *u2 = sgd_uniform(c[2], c[3]);
}

// (sin(pi x), cos(pi x)).  The device has sincospi, whose argument reduction is exact, so no Payne-Hanek table lands in
// local memory; the host reduces x in [0, 2) exactly (Sterbenz) to [0, 1/4] and calls sin / cos there.
SGD_HD void sgd_sincospi(double x, double* s, double* c) {
#if defined(__CUDA_ARCH__)
    sincospi(x, s, c);
#else
    double ss = 1.0, cs = 1.0;
    if (x >= 1.0) { x = x - 1.0; ss = -1.0; cs = -1.0; }                 // sin(pi (x + 1)) = -sin(pi x)
    if (x > 0.5) { x = 1.0 - x; cs = -cs; }                              // sin(pi (1 - x)) = sin, cos flips
    const bool swap = x > 0.25;                                          // sin(pi (1/2 - x)) = cos(pi x)
    if (swap) x = 0.5 - x;
    const double a = sin(M_PI * x), b = cos(M_PI * x);
    *s = ss * (swap ? b : a);
    *c = cs * (swap ? a : b);
#endif
}

// Box-Muller on (u1, u2): r = sqrt(-2 log u1); element 2j is r cos(2 pi u2), element 2j + 1 is r sin(2 pi u2)
SGD_HD void sgd_box_muller(double u1, double u2, double* z0, double* z1) {
    const double r = sgd_sqrt(-2.0 * log(u1));
    double s, c;
    sgd_sincospi(2.0 * u2, &s, &c);
    *z0 = sgd_mul(r, c);
    *z1 = sgd_mul(r, s);
}

// ---- the Adam step -------------------------------------------------------------------------------------------------
// lane l's share of sum_i g_i^2 (i = l, l + SGD_LANES, ... in order) and whether all of them are finite
SGD_HD double sgd_lane_sumsq(const double* g, int n, int lane, bool* finite) {
    double s = 0.0;
    bool f = true;
    for (int i = lane; i < n; i += SGD_LANES) {
        const double x = g[i];
        f = f && isfinite(x);
        s = sgd_add(s, sgd_mul(x, x));
    }
    *finite = f;
    return s;
}

// one level of the lanes' tree: s[l] += s[l + half] for l < half (half = SGD_LANES / 2, ..., 1, in that order)
SGD_HD void sgd_tree_step(double* s, int l, int half) { s[l] = sgd_add(s[l], s[l + half]); }

// the clip scale of a gradient of squared norm ss: max_norm / ||g|| when 0 < max_norm < ||g||, else 1 (no clip)
SGD_HD double sgd_clip_scale(double ss, double max_norm) {
    const double norm = sgd_sqrt(ss);
    return max_norm > 0.0 && norm > max_norm ? sgd_div(max_norm, norm) : 1.0;
}

// one parameter's step with the restart's new running products b1t = b1^t, b2t = b2^t:
//   g <- scale g;  m <- b1 m + (1 - b1) g;  v <- b2 v + (1 - b2) g^2;
//   theta <- theta - lr (m / (1 - b1t)) / (sqrt(v / (1 - b2t)) + eps)
SGD_HD void sgd_adam_elem(double g, double scale, double lr, double b1, double b2, double eps, double b1t, double b2t,
                          double* m, double* v, double* theta) {
    if (scale != 1.0) g = sgd_mul(g, scale);
    const double mm = sgd_add(sgd_mul(b1, *m), sgd_mul(sgd_add(1.0, -b1), g));
    const double vv = sgd_add(sgd_mul(b2, *v), sgd_mul(sgd_add(1.0, -b2), sgd_mul(g, g)));
    const double mh = sgd_div(mm, sgd_add(1.0, -b1t));
    const double vh = sgd_div(vv, sgd_add(1.0, -b2t));
    *m = mm;
    *v = vv;
    *theta = sgd_add(*theta, -sgd_div(sgd_mul(lr, mh), sgd_add(sgd_sqrt(vh), eps)));
}
