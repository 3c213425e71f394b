// rollout_step.cuh -- per-restart device pieces of the forward cascade's step kernels, shared by rollout.cu and the
// noisy cascade (rollout_noise.cu).
#pragma once
#include "rollout.cuh"
#include "small_kernels.cuh"

// squash (optional) + joint, shared by the linear and RBF paths
__device__ __forceinline__ void ro_action_tail(const RoDev& p, int r, const double* mx, const double* sx,
                                               SmallScratch& sc) {
    const int Ds = p.Ds, U = p.U, D = Ds + U;
    const int tid = threadIdx.x, nt = blockDim.x;
    double* Mp = p.Mp + (size_t)r * U;  double* Sp = p.Sp + (size_t)r * U * U;  double* Vp = p.Vp + (size_t)r * Ds * U;
    double* Mu = p.Mu + (size_t)r * U;  double* Su = p.Su + (size_t)r * U * U;
    double* Cq = p.Cq + (size_t)r * U * U;  double* Vu = p.Vu + (size_t)r * Ds * U;
    if (p.squash) {
        dev_squash_sin(U, Mp, Sp, p.maxa, Mu, Su, Cq);
        for (int e = tid; e < Ds * U; e += nt) {
            const int i = e / U, j = e % U;
            double v = 0.0;
            for (int k = 0; k < U; ++k) v = fma(Vp[i * U + k], Cq[k * U + j], v);
            Vu[e] = v;
        }
    } else {
        for (int i = tid; i < U; i += nt) Mu[i] = Mp[i];
        for (int e = tid; e < U * U; e += nt) { Su[e] = Sp[e]; Cq[e] = (e / U == e % U) ? 1.0 : 0.0; }
        for (int e = tid; e < Ds * U; e += nt) Vu[e] = Vp[e];
    }
    __syncthreads();
    dev_joint(Ds, U, mx, sx, Mu, Su, Vu, p.mj + (size_t)r * D, p.sj + (size_t)r * D * D, sc);
}

// cx = [Q, Q V_u],  Q = S_x C^  [Ds, Dh]
__device__ __forceinline__ void tg_cross(const TgDev& g, int r, const double* sx, SmallScratch& sc) {
    const int Ds = g.tm.Ds, Dh = g.p.Ds, U = g.p.U, D = Dh + U;
    const int tid = threadIdx.x, nt = blockDim.x;
    const double* Ch = g.Ch + (size_t)r * Ds * Dh;
    const double* Vu = g.p.Vu + (size_t)r * Dh * U;
    double* cx = g.cx + (size_t)r * Ds * D;
    for (int e = tid; e < Ds * Dh; e += nt) {
        const int i = e / Dh, k = e % Dh;
        double v = 0.0;
        for (int l = 0; l < Ds; ++l) v = fma(sx[i * Ds + l], Ch[l * Dh + k], v);
        sc.C[i * SLD + k] = v;
        cx[i * D + k] = v;
    }
    __syncthreads();
    for (int e = tid; e < Ds * U; e += nt) {
        const int i = e / U, j = e % U;
        double v = 0.0;
        for (int k = 0; k < Dh; ++k) v = fma(sc.C[i * SLD + k], Vu[k * U + j], v);
        cx[i * D + Dh + j] = v;
    }
    __syncthreads();
}
