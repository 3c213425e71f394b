// small_kernels.cuh -- closed-form moment computations done by ONE CTA per rollout (batch element):
// linear policy, sin squashing, joint state/action Gaussian, dynamics glue, rewards.
// All matrices are tiny (<=16x16); inputs/outputs live in global memory, scratch in shared memory.
// Reference: pilco/controllers.py:13-58, pilco/rewards.py:19-61, pilco/models/pilco.py:138-153.
#pragma once
#include "common.cuh"
#include "risk_math.cuh"
#include "trig_math.cuh"

#ifdef __CUDACC__

struct SmallScratch {          // shared-memory scratch for one CTA
    double A[MAXD * SLD];
    double B[MAXD * SLD];
    double C[MAXD * SLD];
    double v[MAXD], w[MAXD];
    int perm[MAXD];
    double det;
};

// LinearController.compute_action without squashing (controllers.py:52-54; conlin.m:57-59)
//   M = W m + b ; S = W s W^T ; V = W^T
__device__ __forceinline__ void dev_linear_action(int Ds, int U, const double* W, const double* b,
                                                  const double* m, const double* s,
                                                  double* Mo, double* So, double* Vo, SmallScratch& sc) {
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int e = tid; e < U * Ds; e += nt) {                 // A = W s   [U,Ds]
        const int i = e / Ds, j = e % Ds;
        double v = 0.0;
        for (int k = 0; k < Ds; ++k) v = fma(W[i * Ds + k], s[k * Ds + j], v);
        sc.A[i * SLD + j] = v;
    }
    for (int i = tid; i < U; i += nt) {
        double v = b[i];
        for (int k = 0; k < Ds; ++k) v = fma(W[i * Ds + k], m[k], v);
        Mo[i] = v;
    }
    for (int e = tid; e < Ds * U; e += nt) { const int i = e / U, j = e % U; Vo[i * U + j] = W[j * Ds + i]; }
    __syncthreads();
    for (int e = tid; e < U * U; e += nt) {
        const int i = e / U, j = e % U;
        double v = 0.0;
        for (int k = 0; k < Ds; ++k) v = fma(sc.A[i * SLD + k], W[j * Ds + k], v);
        So[i * U + j] = v;
    }
    __syncthreads();
}

// squash_sin (controllers.py:13-36; gSin.m:33-48).  In: m[U], s[U,U].  Out: M[U], S[U,U], C[U,U].
// Safe to run in place only if outputs do not alias inputs.
__device__ __forceinline__ void dev_squash_sin(int U, const double* m, const double* s, const double* maxa,
                                               double* Mo, double* So, double* Co) {
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int i = tid; i < U; i += nt) Mo[i] = maxa[i] * exp(-0.5 * s[i * U + i]) * sin(m[i]);
    for (int e = tid; e < U * U; e += nt) {
        const int i = e / U, j = e % U;
        const double lq = -0.5 * (s[i * U + i] + s[j * U + j]);
        const double q = exp(lq);
        const double sij = s[i * U + j];
        const double v = (exp(lq + sij) - q) * cos(m[i] - m[j]) - (exp(lq - sij) - q) * cos(m[i] + m[j]);
        So[e] = 0.5 * maxa[i] * maxa[j] * v;
        Co[e] = (i == j) ? maxa[i] * exp(-0.5 * s[i * U + i]) * cos(m[i]) : 0.0;
    }
    __syncthreads();
}

// joint Gaussian of (x,u) (pilco.py:141-144).  c = inv(s_x) cov(x,u)  [Ds,U].
//   m = [m_x, m_u];  s = [[s_x, s_x c],[ (s_x c)^T, s_u]]
__device__ __forceinline__ void dev_joint(int Ds, int U, const double* mx, const double* sx,
                                          const double* mu, const double* su, const double* c,
                                          double* mj, double* sj, SmallScratch& sc) {
    const int tid = threadIdx.x, nt = blockDim.x, D = Ds + U;
    for (int e = tid; e < Ds * U; e += nt) {                 // A = s_x c
        const int i = e / U, j = e % U;
        double v = 0.0;
        for (int k = 0; k < Ds; ++k) v = fma(sx[i * Ds + k], c[k * U + j], v);
        sc.A[i * SLD + j] = v;
    }
    for (int i = tid; i < D; i += nt) mj[i] = i < Ds ? mx[i] : mu[i - Ds];
    __syncthreads();
    for (int e = tid; e < D * D; e += nt) {
        const int i = e / D, j = e % D;
        double v;
        if (i < Ds && j < Ds) v = sx[i * Ds + j];
        else if (i < Ds) v = sc.A[i * SLD + (j - Ds)];
        else if (j < Ds) v = sc.A[j * SLD + (i - Ds)];
        else v = su[(i - Ds) * U + (j - Ds)];
        sj[e] = v;
    }
    __syncthreads();
}

// next-state glue (pilco.py:147-149):  M_x = M_dx + m_x;  S_x = S_dx + s_x + s1 C + (s1 C)^T,
// s1 = first Ds rows of the joint covariance sj [D,D], C = V_dx [D,Ds].
__device__ __forceinline__ void dev_glue(int Ds, int U, const double* mx, const double* sx, const double* sj,
                                         const double* Md, const double* Sd, const double* Vd,
                                         double* mo, double* so, SmallScratch& sc) {
    const int tid = threadIdx.x, nt = blockDim.x, D = Ds + U;
    for (int e = tid; e < Ds * Ds; e += nt) {
        const int i = e / Ds, j = e % Ds;
        double v = 0.0;
        for (int k = 0; k < D; ++k) v = fma(sj[i * D + k], Vd[k * Ds + j], v);
        sc.A[i * SLD + j] = v;
    }
    __syncthreads();
    for (int i = tid; i < Ds; i += nt) mo[i] = Md[i] + mx[i];
    for (int e = tid; e < Ds * Ds; e += nt) {
        const int i = e / Ds, j = e % Ds;
        so[e] = Sd[e] + sx[e] + sc.A[i * SLD + j] + sc.A[j * SLD + i];
    }
    __syncthreads();
}

// trigonometric feature map of the angular state dimensions (trig_math.cuh): N(m, s) [Ds] -> moments of phi(x) [Dh],
// M [Dh], S [Dh,Dh], C = inv(s) cov(x, phi) [Ds,Dh].  Outputs must not alias inputs.
__device__ __forceinline__ void dev_trig(const TrigMap& tm, const double* m, const double* s,
                                         double* Mo, double* So, double* Co) {
    const int tid = threadIdx.x, nt = blockDim.x, Ds = tm.Ds, Dh = trig_dh(tm);
    for (int k = tid; k < Dh; k += nt) Mo[k] = trig_M_entry(tm, m, s, k);
    for (int e = tid; e < Dh * Dh; e += nt) So[e] = trig_S_entry(tm, m, s, e / Dh, e % Dh);
    for (int e = tid; e < Ds * Dh; e += nt) Co[e] = trig_C_entry(tm, m, s, e / Dh, e % Dh);
    __syncthreads();
}

// VJP of dev_trig: gm [Ds] += d/dm, gs [Ds,Ds] += the symmetric part of d/ds, for cotangents gM, gS, gC (gC may be NULL)
__device__ __forceinline__ void dev_trig_bwd(const TrigMap& tm, const double* m, const double* s, const double* gM,
                                             const double* gS, const double* gC, double* gm, double* gs) {
    const int tid = threadIdx.x, nt = blockDim.x, Ds = tm.Ds;
    for (int i = tid; i < Ds; i += nt) gm[i] += trig_vjp_m(tm, m, s, gM, gS, gC, i);
    for (int e = tid; e < Ds * Ds; e += nt) gs[e] += trig_vjp_s(tm, m, s, gM, gS, gC, e / Ds, e % Ds);
    __syncthreads();
}

// ExponentialReward (rewards.py:19-51; reward.m:35-57):
//   muR = exp(-0.5 (m-t)^T W (I+sW)^-1 (m-t)) / sqrt(det(I+sW));  r2 likewise with 2 s W;  sR = r2 - muR^2
// Returns muR to every thread; *sR_out written by thread 0 when non-null.
__device__ __forceinline__ double dev_exp_reward(int Ds, const double* W, const double* t,
                                                 const double* m, const double* s,
                                                 double* sR_out, SmallScratch& sc) {
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
    double mu = 0.0, r2 = 0.0;
    const int npass = sR_out ? 2 : 1;
    for (int pass = 0; pass < npass; ++pass) {
        const double f = pass == 0 ? 1.0 : 2.0;
        __syncthreads();
        for (int e = tid; e < Ds * Ds; e += nt) {            // A = I + f s W
            const int i = e / Ds, j = e % Ds;
            double v = 0.0;
            for (int k = 0; k < Ds; ++k) v = fma(s[i * Ds + k], W[k * Ds + j], v);
            sc.A[i * SLD + j] = f * v + (i == j ? 1.0 : 0.0);
        }
        for (int i = tid; i < Ds; i += nt) { sc.v[i] = m[i] - t[i]; sc.B[i * SLD] = m[i] - t[i]; }
        __syncthreads();
        if (warp == 0) {
            double det;
            lu_warp(sc.A, sc.perm, Ds, lane, &det);
            lu_solve_warp(sc.A, sc.perm, sc.B, sc.C, Ds, 1, lane);   // C[:,0] = (I+fsW)^-1 (m-t)
            if (lane == 0) sc.det = det;
        }
        __syncthreads();
        // quad = (m-t)^T W y
        double quad = 0.0;
        for (int i = 0; i < Ds; ++i) {
            double wy = 0.0;
            for (int k = 0; k < Ds; ++k) wy = fma(W[i * Ds + k], sc.C[k * SLD], wy);
            quad = fma(sc.v[i], wy, quad);
        }
        const double val = exp(-0.5 * f * quad) / sqrt(sc.det);
        if (pass == 0) mu = val; else r2 = val;
    }
    if (sR_out && tid == 0) *sR_out = r2 - mu * mu;
    __syncthreads();
    return mu;
}

// LinearReward (rewards.py:53-61): muR = m . W ; sR = W^T s W
__device__ __forceinline__ double dev_linear_reward(int Ds, const double* W, const double* m, const double* s,
                                                    double* sR_out) {
    double mu = 0.0;
    for (int i = 0; i < Ds; ++i) mu = fma(m[i], W[i], mu);
    if (sR_out && threadIdx.x == 0) {
        double v = 0.0;
        for (int i = 0; i < Ds; ++i) for (int j = 0; j < Ds; ++j) v = fma(W[i] * s[i * Ds + j], W[j], v);
        *sR_out = v;
    }
    return mu;
}

// Expected value of one reward term at the state moments (m, s); every thread gets the value.
__device__ __forceinline__ double dev_reward_value(int Ds, const pilco_reward_term& rt, const double* m, const double* s,
                                                   SmallScratch& sc) {
    if (rt.kind == PILCO_REWARD_EXP) return dev_exp_reward(Ds, rt.W, rt.t, m, s, nullptr, sc);
    if (rt.kind == PILCO_REWARD_BOX) return risk_box_eval(Ds, rt.W, m, s, nullptr, nullptr);
    return dev_linear_reward(Ds, rt.W, m, s, nullptr);
}

// Expected value of one term on the joint state-action Gaussian (PILCO_REWARD_*_SA) at its moments (m, s) of dimension
// D = Ds + U: the same closed forms (SmallScratch holds MAXD x SLD either way); every thread gets the value.
__device__ __forceinline__ double dev_joint_reward_value(int D, const pilco_reward_term& rt, const double* m, const double* s,
                                                         SmallScratch& sc) {
    if (rt.kind == PILCO_REWARD_EXP_SA) return dev_exp_reward(D, rt.W, rt.t, m, s, nullptr, sc);
    return dev_linear_reward(D, rt.W, m, s, nullptr);
}

// ---------------------------------------------------------------------------------------------
// VJPs (numpy statement: oracle/staged.py).  All "g*" outputs marked += accumulate.
// ---------------------------------------------------------------------------------------------
// squash_sin VJP.  m,s: pre-squash moments; Mu,Su: squashed outputs; gM,gS,gCd: upstream cotangents of
// (M, S, diag C).  Writes gm[U], gs[U,U].
__device__ __forceinline__ void dev_squash_bwd(int U, const double* m, const double* s, const double* maxa,
                                               const double* Mu, const double* Su,
                                               const double* gM, const double* gS, const double* gCd,
                                               double* gm, double* gs) {
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int e = tid; e < U * U; e += nt) {
        const int i = e / U, j = e % U;
        const double lq = -0.5 * (s[i * U + i] + s[j * U + j]);
        const double E1 = exp(lq + s[e]), E2 = exp(lq - s[e]);
        gs[e] = gS[e] * 0.5 * maxa[i] * maxa[j] * (E1 * cos(m[i] - m[j]) + E2 * cos(m[i] + m[j]));
    }
    __syncthreads();
    for (int i = tid; i < U; i += nt) {
        const double ci = maxa[i] * exp(-0.5 * s[i * U + i]) * cos(m[i]);
        double gmi = gM[i] * ci - gCd[i] * Mu[i];
        double gd = -0.5 * gM[i] * Mu[i] - 0.5 * gCd[i] * ci;
        for (int j = 0; j < U; ++j) {
            const double lq = -0.5 * (s[i * U + i] + s[j * U + j]);
            const double q = exp(lq);
            const double f = 0.5 * maxa[i] * maxa[j];
            const double sij = s[i * U + j], sji = s[j * U + i];
            // pair (i,j): derivative w.r.t. m_i (first index)
            gmi += gS[i * U + j] * f * (-(exp(lq + sij) - q) * sin(m[i] - m[j]) + (exp(lq - sij) - q) * sin(m[i] + m[j]));
            // pair (j,i): derivative w.r.t. m_i (second index)
            gmi += gS[j * U + i] * f * ((exp(lq + sji) - q) * sin(m[j] - m[i]) + (exp(lq - sji) - q) * sin(m[j] + m[i]));
            gd += -0.5 * (gS[i * U + j] * Su[i * U + j] + gS[j * U + i] * Su[j * U + i]);
        }
        gm[i] = gmi;
        gs[i * U + i] += gd;
    }
    __syncthreads();
}

// ExponentialReward VJP (reward.m:48-49, W symmetric):  gm += scale dmu/dm,  gS += scale dmu/dS
__device__ __forceinline__ void dev_exp_reward_bwd(int Ds, const double* W, const double* t, const double* m,
                                                   const double* s, double scale, double* gm, double* gS,
                                                   SmallScratch& sc) {
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
    __syncthreads();
    for (int e = tid; e < Ds * Ds; e += nt) {
        const int i = e / Ds, j = e % Ds;
        double v = 0.0;
        for (int k = 0; k < Ds; ++k) v = fma(s[i * Ds + k], W[k * Ds + j], v);
        sc.A[i * SLD + j] = v + (i == j ? 1.0 : 0.0);
        sc.B[i * SLD + j] = (i == j) ? 1.0 : 0.0;
    }
    for (int i = tid; i < Ds; i += nt) sc.v[i] = m[i] - t[i];
    __syncthreads();
    if (warp == 0) {
        double det;
        lu_warp(sc.A, sc.perm, Ds, lane, &det);
        lu_solve_warp(sc.A, sc.perm, sc.B, sc.C, Ds, Ds, lane);          // C = (I + sW)^-1
        if (lane == 0) sc.det = det;
    }
    __syncthreads();
    for (int e = tid; e < Ds * Ds; e += nt) {                            // B = iSpW = W (I+sW)^-1
        const int i = e / Ds, j = e % Ds;
        double v = 0.0;
        for (int k = 0; k < Ds; ++k) v = fma(W[i * Ds + k], sc.C[k * SLD + j], v);
        sc.B[i * SLD + j] = v;
    }
    __syncthreads();
    for (int i = tid; i < Ds; i += nt) {
        double v = 0.0;
        for (int k = 0; k < Ds; ++k) v = fma(sc.B[i * SLD + k], sc.v[k], v);
        sc.w[i] = v;                                                     // wy = iSpW (m-t)
    }
    __syncthreads();
    double quad = 0.0;
    for (int i = 0; i < Ds; ++i) quad = fma(sc.v[i], sc.w[i], quad);
    const double mu = exp(-0.5 * quad) / sqrt(sc.det);
    for (int i = tid; i < Ds; i += nt) gm[i] += -scale * mu * sc.w[i];
    for (int e = tid; e < Ds * Ds; e += nt) {
        const int i = e / Ds, j = e % Ds;
        const double isym = 0.5 * (sc.B[i * SLD + j] + sc.B[j * SLD + i]);
        gS[e] += 0.5 * scale * mu * (sc.w[i] * sc.w[j] - isym);
    }
    __syncthreads();
}

// VJP of a power of the f-scaled ExponentialReward moment (reward.m:52-66: f = 1 the mean, f = 2 the second moment)
//   r_f = exp(-f/2 (m-t)^T W (I+f sW)^-1 (m-t)) / sqrt(det(I+f sW)),  w_f = W (I+f sW)^-1 (m-t):
//   d r_f/dm = -f r_f w_f,  d r_f/dS = (f/2) r_f (f w_f w_f^T - W (I+f sW)^-1)
// gm += scale d(r_f^p)/dm, gS += scale d(r_f^p)/dS (p = 1 or 2), symmetrised as dev_exp_reward_bwd; returns r_f.
__device__ __forceinline__ double dev_exp_moment_bwd(int Ds, const double* W, const double* t, const double* m,
                                                     const double* s, double f, int p, double scale, double* gm,
                                                     double* gS, SmallScratch& sc) {
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
    __syncthreads();
    for (int e = tid; e < Ds * Ds; e += nt) {
        const int i = e / Ds, j = e % Ds;
        double v = 0.0;
        for (int k = 0; k < Ds; ++k) v = fma(s[i * Ds + k], W[k * Ds + j], v);
        sc.A[i * SLD + j] = f * v + (i == j ? 1.0 : 0.0);
        sc.B[i * SLD + j] = (i == j) ? 1.0 : 0.0;
    }
    for (int i = tid; i < Ds; i += nt) sc.v[i] = m[i] - t[i];
    __syncthreads();
    if (warp == 0) {
        double det;
        lu_warp(sc.A, sc.perm, Ds, lane, &det);
        lu_solve_warp(sc.A, sc.perm, sc.B, sc.C, Ds, Ds, lane);          // C = (I + f sW)^-1
        if (lane == 0) sc.det = det;
    }
    __syncthreads();
    for (int e = tid; e < Ds * Ds; e += nt) {                            // B = W (I + f sW)^-1
        const int i = e / Ds, j = e % Ds;
        double v = 0.0;
        for (int k = 0; k < Ds; ++k) v = fma(W[i * Ds + k], sc.C[k * SLD + j], v);
        sc.B[i * SLD + j] = v;
    }
    __syncthreads();
    for (int i = tid; i < Ds; i += nt) {
        double v = 0.0;
        for (int k = 0; k < Ds; ++k) v = fma(sc.B[i * SLD + k], sc.v[k], v);
        sc.w[i] = v;
    }
    __syncthreads();
    double quad = 0.0;
    for (int i = 0; i < Ds; ++i) quad = fma(sc.v[i], sc.w[i], quad);
    const double rf = exp(-0.5 * f * quad) / sqrt(sc.det);
    const double c = (p == 2 ? 2.0 * rf : 1.0) * scale * rf;              // scale d(r_f^p)/d r_f times r_f
    for (int i = tid; i < Ds; i += nt) gm[i] += -f * c * sc.w[i];
    for (int e = tid; e < Ds * Ds; e += nt) {
        const int i = e / Ds, j = e % Ds;
        const double isym = 0.5 * (sc.B[i * SLD + j] + sc.B[j * SLD + i]);
        gS[e] += 0.5 * f * c * (f * sc.w[i] * sc.w[j] - isym);
    }
    __syncthreads();
    return rf;
}

// LinearController VJP: gW += gMp m^T + (gSp+gSp^T) W s + gVp^T ; gb += gMp ; gm += W^T gMp ; gS += W^T gSp W
__device__ __forceinline__ void dev_linear_bwd(int Ds, int U, const double* W, const double* m, const double* s,
                                               const double* gMp, const double* gSp, const double* gVp,
                                               double* gW, double* gb, double* gm, double* gS, SmallScratch& sc) {
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int e = tid; e < U * Ds; e += nt) {                 // A = W s  [U,Ds]
        const int i = e / Ds, k = e % Ds;
        double v = 0.0;
        for (int l = 0; l < Ds; ++l) v = fma(W[i * Ds + l], 0.5 * (s[l * Ds + k] + s[k * Ds + l]), v);
        sc.A[i * SLD + k] = v;
    }
    for (int e = tid; e < U * Ds; e += nt) {                 // B = gSp W  [U,Ds]
        const int i = e / Ds, k = e % Ds;
        double v = 0.0;
        for (int j = 0; j < U; ++j) v = fma(gSp[i * U + j], W[j * Ds + k], v);
        sc.B[i * SLD + k] = v;
    }
    __syncthreads();
    for (int e = tid; e < U * Ds; e += nt) {
        const int i = e / Ds, k = e % Ds;
        double v = gMp[i] * m[k] + gVp[k * U + i];
        for (int j = 0; j < U; ++j) v = fma(gSp[i * U + j] + gSp[j * U + i], sc.A[j * SLD + k], v);
        gW[e] += v;
    }
    for (int i = tid; i < U; i += nt) gb[i] += gMp[i];
    for (int k = tid; k < Ds; k += nt) {
        double v = 0.0;
        for (int i = 0; i < U; ++i) v = fma(W[i * Ds + k], gMp[i], v);
        gm[k] += v;
    }
    for (int e = tid; e < Ds * Ds; e += nt) {
        const int k = e / Ds, l = e % Ds;
        double v = 0.0;
        for (int i = 0; i < U; ++i) v = fma(W[i * Ds + k], sc.B[i * SLD + l], v);
        gS[e] += v;
    }
    __syncthreads();
}

// Box-risk VJP (safe_pilco_extension/rewards_safe.py:13-58; formulas in risk_math.cuh):
//   gm[d] += scale d risk/d m[d],  gS[d,d] += scale d risk/d s[d,d]   for the constrained dimensions
__device__ __forceinline__ void dev_box_risk_bwd(int Ds, const double* prm, const double* m, const double* s,
                                                 double scale, double* gm, double* gS) {
    if (threadIdx.x == 0) {
        double dm[RISK_MAX_DIMS], dv[RISK_MAX_DIMS];
        risk_box_eval(Ds, prm, m, s, dm, dv);
        const int nd = (int)prm[0];
        for (int k = 0; k < nd; ++k) {
            const int d = (int)prm[3 + 3 * k];
            gm[d] += scale * dm[k];
            gS[d * Ds + d] += scale * dv[k];
        }
    }
    __syncthreads();
}

// VJP of one reward term with upstream weight `scale` (accumulates into gm, gS)
__device__ __forceinline__ void dev_reward_bwd(int Ds, const pilco_reward_term& rt, const double* m, const double* s,
                                               double scale, double* gm, double* gS, SmallScratch& sc) {
    if (rt.kind == PILCO_REWARD_EXP) dev_exp_reward_bwd(Ds, rt.W, rt.t, m, s, scale, gm, gS, sc);
    else if (rt.kind == PILCO_REWARD_BOX) dev_box_risk_bwd(Ds, rt.W, m, s, scale, gm, gS);
    else {
        for (int i = threadIdx.x; i < Ds; i += blockDim.x) gm[i] += scale * rt.W[i];
        __syncthreads();
    }
}

// VJP of one joint state-action term (dev_joint_reward_value) with upstream weight `scale` (accumulates into gm, gS)
__device__ __forceinline__ void dev_joint_reward_bwd(int D, const pilco_reward_term& rt, const double* m, const double* s,
                                                     double scale, double* gm, double* gS, SmallScratch& sc) {
    if (rt.kind == PILCO_REWARD_EXP_SA) dev_exp_reward_bwd(D, rt.W, rt.t, m, s, scale, gm, gS, sc);
    else {
        for (int i = threadIdx.x; i < D; i += blockDim.x) gm[i] += scale * rt.W[i];
        __syncthreads();
    }
}

#endif  // __CUDACC__
