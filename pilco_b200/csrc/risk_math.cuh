// risk_math.cuh -- closed-form "probability of lying in a box" reward of the safe-PILCO extension and its
// derivatives.  Plain scalar code, usable from device code and (for the CPU unit test of the formulas,
// tests/test_host.py) from a host compiler.
//
// Reference: safe_pilco_extension/rewards_safe.py:13-58.  Both reward classes evaluate, per constrained state
// dimension d, a univariate normal with loc = m[d] and   scale = sfac * s[d,d]   (the reference passes the
// VARIANCE entry -- twice it for RiskOfCollision, rewards_safe.py:21 -- as tfd.Normal's `scale`; reproduced
// as written) and multiply the per-dimension interval probabilities:
//   RiskOfCollision (rewards_safe.py:20-25): dims (0, 2), sfac = 2, both bounds, inside
//   SingleConstraint (rewards_safe.py:44-58): one dim, sfac = 1, optional bounds, optional complement
//
// Parameter block `prm` (doubles): [nd, inside, sfac, (dim_k, low_k, high_k) x nd]; a missing bound is +-inf.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define RISK_HD __host__ __device__ __forceinline__
#else
#define RISK_HD inline
#endif

#define RISK_MAX_DIMS 16
#define RISK_PRM_LEN(nd) (3 + 3 * (nd))

RISK_HD double risk_Phi(double x) { return 0.5 * erfc(-x * 0.70710678118654752440); }
RISK_HD double risk_phi(double x) { return 0.39894228040143267794 * exp(-0.5 * x * x); }

// value of the box probability; when dm != nullptr also d value / d m[dim_k] -> dm[k] and
// d value / d s[dim_k, dim_k] -> dv[k]  (k < nd).  Returns NaN-free results for infinite bounds.
RISK_HD double risk_box_eval(int Ds, const double* prm, const double* m, const double* s, double* dm, double* dv) {
    const int nd = (int)prm[0];
    const bool inside = prm[1] != 0.0;
    const double sfac = prm[2];
    double F[RISK_MAX_DIMS], Fm[RISK_MAX_DIMS], Fv[RISK_MAX_DIMS];
    for (int k = 0; k < nd; ++k) {
        const int d = (int)prm[3 + 3 * k];
        const double lo = prm[4 + 3 * k], hi = prm[5 + 3 * k];
        const double sig = sfac * s[d * Ds + d];
        const double mu = m[d];
        double Ph = 1.0, ph = 0.0, bph = 0.0, Pl = 0.0, pl = 0.0, apl = 0.0;
        if (hi < 1e300) { const double b = (hi - mu) / sig; Ph = risk_Phi(b); ph = risk_phi(b); bph = b * ph; }
        if (lo > -1e300) { const double a = (lo - mu) / sig; Pl = risk_Phi(a); pl = risk_phi(a); apl = a * pl; }
        F[k] = Ph - Pl;
        Fm[k] = -(ph - pl) / sig;                  // d/d mu
        Fv[k] = -(bph - apl) / sig * sfac;         // d/d s[d,d] = d/d sig * sfac
    }
    double val = 1.0;
    for (int k = 0; k < nd; ++k) val *= F[k];
    if (dm) {
        for (int k = 0; k < nd; ++k) {
            double rest = 1.0;
            for (int j = 0; j < nd; ++j) if (j != k) rest *= F[j];
            dm[k] = (inside ? 1.0 : -1.0) * rest * Fm[k];
            dv[k] = (inside ? 1.0 : -1.0) * rest * Fv[k];
        }
    }
    return inside ? val : 1.0 - val;
}

// the same box at a point x (risk_box_eval as s -> 0, used by the particle rollout): the indicator that every
// constrained dimension lies strictly inside (low_k, high_k), complemented when inside = 0
RISK_HD double risk_box_point(const double* prm, const double* x) {
    const int nd = (int)prm[0];
    const bool inside = prm[1] != 0.0;
    bool in = true;
    for (int k = 0; k < nd; ++k) {
        const double v = x[(int)prm[3 + 3 * k]];
        in = in && prm[4 + 3 * k] < v && v < prm[5 + 3 * k];
    }
    return (in == inside) ? 1.0 : 0.0;
}
