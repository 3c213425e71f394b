// trig_math.cuh -- closed-form moments of the trigonometric feature map of angular state dimensions (PILCO's gTrig
// inside propagate.m) and their VJP.  Plain scalar code, usable from device code and (for the CPU unit test of the
// formulas, tests/test_angles_host.py) from a host compiler.
//
// State x [Ds] ~ N(m, s) with angular dimensions a_1 .. a_A.  The feature map
//   phi(x) = [x_j for j not an angle, increasing j] ++ [sin x_a1, cos x_a1, ..., sin x_aA, cos x_aA]     (Dh = Ds + A)
// has the exact moments
//   E[sin x_a] = exp(-s_aa/2) sin m_a,   E[cos x_a] = exp(-s_aa/2) cos m_a,
//   cov(x_j, sin x_a) = s_ja E[cos x_a],  cov(x_j, cos x_a) = -s_ja E[sin x_a],
// and, between angles a and b (a = b included) with q = exp(-(s_aa + s_bb)/2), u = expm1(s_ab), v = expm1(-s_ab),
//   cov(sin a, sin b) = q/2 (u cos(m_a - m_b) - v cos(m_a + m_b))      cov(sin a, cos b) = q/2 (v sin(m_a + m_b) + u sin(m_a - m_b))
//   cov(cos a, cos b) = q/2 (u cos(m_a - m_b) + v cos(m_a + m_b))      cov(cos a, sin b) = q/2 (v sin(m_a + m_b) - u sin(m_a - m_b))
// (the e+- = q exp(-+s_ab) products of the second moments minus the products of the means, written with expm1 so
// that small covariances do not cancel).  The cross factor C = inv(s) cov(x, phi) [Ds, Dh] needs no inverse:
// e_j for a pass-through column, E[cos x_a] e_a for the sine column of angle a, -E[sin x_a] e_a for its cosine column.
//
// Entry (k, l) of the output covariance reads s[i][j] in that orientation (i, j the state dimensions of k and l); the
// VJP returns the symmetric part of the resulting gradient with respect to s.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define TRIG_HD __host__ __device__ __forceinline__
#else
#define TRIG_HD inline
#endif

#define TRIG_MAX 16

struct TrigMap {
    int Ds, A, np;              // state dimension, number of angles, number of pass-through dimensions (Ds - A)
    int pass[TRIG_MAX];         // pass-through state dimensions, increasing
    int ang[TRIG_MAX];          // angular state dimensions, in the caller's order
    int pos[TRIG_MAX];          // state dimension -> its feature column (an angle: its sine column)
    int isang[TRIG_MAX];        // state dimension -> 1 + its angle index, 0 for a pass-through dimension
};

// Build the map; nonzero when A is outside [0, Ds], Ds outside [1, TRIG_MAX], or an index is out of range or repeated.
TRIG_HD int trig_map_make(int Ds, int A, const int* dims, TrigMap* tm) {
    if (Ds < 1 || Ds > TRIG_MAX || A < 0 || A > Ds) return 1;
    tm->Ds = Ds; tm->A = A; tm->np = Ds - A;
    for (int i = 0; i < TRIG_MAX; ++i) { tm->isang[i] = 0; tm->pos[i] = 0; tm->pass[i] = 0; tm->ang[i] = 0; }
    for (int i = 0; i < A; ++i) {
        const int d = dims[i];
        if (d < 0 || d >= Ds || tm->isang[d]) return 1;
        tm->isang[d] = 1 + i; tm->ang[i] = d; tm->pos[d] = Ds - A + 2 * i;
    }
    int k = 0;
    for (int d = 0; d < Ds; ++d) if (!tm->isang[d]) { tm->pass[k] = d; tm->pos[d] = k; ++k; }
    return 0;
}

TRIG_HD int trig_dh(const TrigMap& tm) { return tm.Ds + tm.A; }

// feature column k -> state dimension and kind (0: pass-through, 1: sine, 2: cosine)
TRIG_HD void trig_col(const TrigMap& tm, int k, int* dim, int* kind) {
    if (k < tm.np) { *dim = tm.pass[k]; *kind = 0; }
    else { const int i = (k - tm.np) >> 1; *dim = tm.ang[i]; *kind = 1 + ((k - tm.np) & 1); }
}

TRIG_HD void trig_mean(double m, double saa, double* es, double* ec) {
    const double e = exp(-0.5 * saa);
    *es = e * sin(m); *ec = e * cos(m);
}

// covariance block of the angle pair (a, b): c = [cov(sin a, sin b), cov(sin a, cos b), cov(cos a, sin b), cov(cos a, cos b)]
TRIG_HD void trig_pair_cov(double ma, double mb, double saa, double sbb, double sab, double* c) {
    const double h = 0.5 * exp(-0.5 * (saa + sbb)), u = expm1(sab), v = expm1(-sab);
    const double cm = cos(ma - mb), cp = cos(ma + mb), sm = sin(ma - mb), sp = sin(ma + mb);
    c[0] = h * (u * cm - v * cp);
    c[1] = h * (v * sp + u * sm);
    c[2] = h * (v * sp - u * sm);
    c[3] = h * (u * cm + v * cp);
}

// VJP of trig_pair_cov with cotangent g[4]: d = [d/dma, d/dmb, d/dsaa, d/dsbb, d/dsab]
TRIG_HD void trig_pair_cov_vjp(double ma, double mb, double saa, double sbb, double sab, const double* g, double* d) {
    const double h = 0.5 * exp(-0.5 * (saa + sbb)), u = expm1(sab), v = expm1(-sab), u1 = u + 1.0, v1 = v + 1.0;
    const double cm = cos(ma - mb), cp = cos(ma + mb), sm = sin(ma - mb), sp = sin(ma + mb);
    const double c0 = h * (u * cm - v * cp), c1 = h * (v * sp + u * sm), c2 = h * (v * sp - u * sm), c3 = h * (u * cm + v * cp);
    d[0] = h * (g[0] * (v * sp - u * sm) + g[1] * (v * cp + u * cm) + g[2] * (v * cp - u * cm) + g[3] * (-u * sm - v * sp));
    d[1] = h * (g[0] * (u * sm + v * sp) + g[1] * (v * cp - u * cm) + g[2] * (v * cp + u * cm) + g[3] * (u * sm - v * sp));
    d[2] = d[3] = -0.5 * (g[0] * c0 + g[1] * c1 + g[2] * c2 + g[3] * c3);
    d[4] = h * (g[0] * (u1 * cm + v1 * cp) + g[1] * (u1 * sm - v1 * sp) - g[2] * (v1 * sp + u1 * sm) + g[3] * (u1 * cm - v1 * cp));
}

// ---- forward, one output entry each ----------------------------------------------------------------------------
TRIG_HD double trig_M_entry(const TrigMap& tm, const double* m, const double* s, int k) {
    int d, kind;
    trig_col(tm, k, &d, &kind);
    if (kind == 0) return m[d];
    double es, ec;
    trig_mean(m[d], s[d * tm.Ds + d], &es, &ec);
    return kind == 1 ? es : ec;
}

TRIG_HD double trig_S_entry(const TrigMap& tm, const double* m, const double* s, int k, int l) {
    const int Ds = tm.Ds;
    int i, ki, j, kj;
    trig_col(tm, k, &i, &ki);
    trig_col(tm, l, &j, &kj);
    if (ki == 0 && kj == 0) return s[i * Ds + j];
    if (ki == 0 || kj == 0) {                  // pass-through dimension x against a trigonometric feature of angle a
        const int a = ki == 0 ? j : i, kind = ki == 0 ? kj : ki;
        double es, ec;
        trig_mean(m[a], s[a * Ds + a], &es, &ec);
        return s[i * Ds + j] * (kind == 1 ? ec : -es);
    }
    double c[4];
    trig_pair_cov(m[i], m[j], s[i * Ds + i], s[j * Ds + j], s[i * Ds + j], c);
    return ki == 1 ? (kj == 1 ? c[0] : c[1]) : (kj == 1 ? c[2] : c[3]);
}

TRIG_HD double trig_C_entry(const TrigMap& tm, const double* m, const double* s, int i, int k) {
    int d, kind;
    trig_col(tm, k, &d, &kind);
    if (d != i) return 0.0;
    if (kind == 0) return 1.0;
    double es, ec;
    trig_mean(m[d], s[d * tm.Ds + d], &es, &ec);
    return kind == 1 ? ec : -es;
}

// ---- VJP: (gM [Dh], gS [Dh,Dh], gC [Ds,Dh] or NULL) -> one entry of gm [Ds] / of the symmetric gs [Ds,Ds] ------------
// cotangents of E[sin x_a], E[cos x_a] gathered from the means, the cross factor and the pass-through cross covariances
TRIG_HD void trig_mean_cot(const TrigMap& tm, const double* s, const double* gM, const double* gS, const double* gC,
                           int a, double* g_es, double* g_ec) {
    const int Ds = tm.Ds, Dh = trig_dh(tm), ks = tm.pos[a], kc = ks + 1;
    double ges = gM[ks], gec = gM[kc];
    if (gC) { gec += gC[a * Dh + ks]; ges -= gC[a * Dh + kc]; }
    for (int q = 0; q < tm.np; ++q) {
        const int j = tm.pass[q];
        gec += gS[q * Dh + ks] * s[j * Ds + a] + gS[ks * Dh + q] * s[a * Ds + j];
        ges -= gS[q * Dh + kc] * s[j * Ds + a] + gS[kc * Dh + q] * s[a * Ds + j];
    }
    *g_es = ges; *g_ec = gec;
}

// d/d(ma, mb, saa, sbb, sab) of the 2 x 2 block of the angle pair (a, b) (state dimensions) under gS
TRIG_HD void trig_pair_grad(const TrigMap& tm, const double* m, const double* s, const double* gS, int a, int b, double* d) {
    const int Ds = tm.Ds, Dh = trig_dh(tm), ka = tm.pos[a], kb = tm.pos[b];
    const double g[4] = {gS[ka * Dh + kb], gS[ka * Dh + kb + 1], gS[(ka + 1) * Dh + kb], gS[(ka + 1) * Dh + kb + 1]};
    trig_pair_cov_vjp(m[a], m[b], s[a * Ds + a], s[b * Ds + b], s[a * Ds + b], g, d);
}

TRIG_HD double trig_vjp_m(const TrigMap& tm, const double* m, const double* s, const double* gM, const double* gS,
                          const double* gC, int i) {
    if (!tm.isang[i]) return gM[tm.pos[i]];
    const int Ds = tm.Ds;
    double ges, gec, es, ec, d[5];
    trig_mean_cot(tm, s, gM, gS, gC, i, &ges, &gec);
    trig_mean(m[i], s[i * Ds + i], &es, &ec);
    double v = ges * ec - gec * es;
    for (int q = 0; q < tm.A; ++q) {
        const int b = tm.ang[q];
        trig_pair_grad(tm, m, s, gS, i, b, d); v += d[0];
        trig_pair_grad(tm, m, s, gS, b, i, d); v += d[1];
    }
    return v;
}

TRIG_HD double trig_vjp_s(const TrigMap& tm, const double* m, const double* s, const double* gM, const double* gS,
                          const double* gC, int i, int j) {
    const int Ds = tm.Ds, Dh = trig_dh(tm), ai = tm.isang[i], aj = tm.isang[j], ki = tm.pos[i], kj = tm.pos[j];
    if (!ai && !aj) return 0.5 * (gS[ki * Dh + kj] + gS[kj * Dh + ki]);
    if (!ai || !aj) {                                  // pass-through p against angle a
        const int p = ai ? j : i, a = ai ? i : j, kp = tm.pos[p], ka = tm.pos[a];
        double es, ec;
        trig_mean(m[a], s[a * Ds + a], &es, &ec);
        return 0.5 * (ec * (gS[kp * Dh + ka] + gS[ka * Dh + kp]) - es * (gS[kp * Dh + ka + 1] + gS[(ka + 1) * Dh + kp]));
    }
    double d[5];
    if (i != j) {
        double v;
        trig_pair_grad(tm, m, s, gS, i, j, d); v = d[4];
        trig_pair_grad(tm, m, s, gS, j, i, d); v += d[4];
        return 0.5 * v;
    }
    double ges, gec, es, ec;
    trig_mean_cot(tm, s, gM, gS, gC, i, &ges, &gec);
    trig_mean(m[i], s[i * Ds + i], &es, &ec);
    double v = -0.5 * (ges * es + gec * ec);
    for (int q = 0; q < tm.A; ++q) {
        const int b = tm.ang[q];
        trig_pair_grad(tm, m, s, gS, i, b, d); v += d[2] + (b == i ? d[4] : 0.0);
        trig_pair_grad(tm, m, s, gS, b, i, d); v += d[3];
    }
    return v;
}
