// rollout_noise.cu -- measurement noise at the policy's input on the moment-matching rollout (pilco_rollout_noisy_*):
// propagate.m's noisy state measurement, ss = S + diag(sn2) for the policy and q = S(j,i) C for the joint.
// The cascade is the one on phi (rollout.cu, rollout_bwd.cu; with no angles phi is the identity and A = 0) with two
// kernels replaced per step:
//   forward  nz_state<t> in place of tg_state: the glue, then the feature moments twice, (m^_x, S^_x, C^_x) under
//            N(m, S) for the dynamics and (m^_z, S^_z) under N(m, S + diag(v)) for the policy (kept per step for the
//            reverse sweep); linear policy at the noisy set, squash, the joint [phi, u] and cx at the true set.  The
//            RBF policy's moment match reads the noisy slots; tg_policy, the dynamics and the reward launches (with
//            exploration, its launches too) are those of the angle / exploration calls.
//   reverse  tg_post (or the taped tg_dyn_finish) without its linear-policy VJP; the RBF policy's VJP reads the noisy
//            slots and accumulates into (gm^_z, gS^_z); nz_trig in place of tg_trig: the linear-policy VJP at the noisy
//            set into (gm^_z, gS^_z), dev_trig_bwd at (m, S) with (gm^_x, gS^_x, gC^_x) and at (m, S + diag(v)) with
//            (gm^_z, gS^_z, 0) into (gm, gS) (dS_z / dS = I), then tg_trig's reward gradients and seeds of step t-1.
// A translation unit of its own, so that the existing kernels compile exactly as they do without it.
#include <cmath>

#include "rollout_bwd.cuh"
#include "rollout_step.cuh"
#include "small_kernels.cuh"

struct NzDev {
    TgDev g;
    double *mz, *Sz;                  // noisy feature moments of step t [R, Dh], [R, Dh, Dh]
    double var[MAXD];
};

struct NzBwdDev {
    TbDev g;
    const double *mz, *Sz;            // forward's noisy feature moments of step t
    double *gmz, *gSz;                // their cotangent [R, Dh], [R, Dh, Dh]
    double var[MAXD];
};

// sn = s + diag(var) in shared memory [Ds, Ds]
__device__ __forceinline__ void nz_noisy_cov(int Ds, const double* s, const double* var, double* sn) {
    for (int e = threadIdx.x; e < Ds * Ds; e += blockDim.x) {
        const int i = e / Ds, j = e % Ds;
        sn[e] = i == j ? s[e] + var[i] : s[e];
    }
    __syncthreads();
}

__global__ void __launch_bounds__(128) nz_state_kernel(NzDev z) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    __shared__ double sn[TRIG_MAX * TRIG_MAX];
    const TgDev& g = z.g;
    const RoDev& p = g.p;
    const int r = blockIdx.x, t = p.t, Ds = g.tm.Ds, Dh = p.Ds, U = p.U;
    const int tid = threadIdx.x, nt = blockDim.x;
    double* mx = p.traj_m + ((size_t)r * (p.H + 1) + t) * Ds;
    double* sx = p.traj_S + ((size_t)r * (p.H + 1) + t) * Ds * Ds;
    if (t == 0) {
        for (int i = tid; i < Ds; i += nt) mx[i] = p.m0[(size_t)r * p.m0_bs + i];
        for (int e = tid; e < Ds * Ds; e += nt) sx[e] = p.S0[(size_t)r * p.S0_bs + e];
        __syncthreads();
    } else {
        mm_finish_device(p.dyn_prev, r);
        __syncthreads();
        const int D = Dh + U;                          // the glue with cx, as tg_state
        dev_glue(Ds, D - Ds, mx - Ds, sx - Ds * Ds, g.cx_prev + (size_t)r * Ds * D,
                 p.Md_prev + (size_t)r * Ds, p.Sd_prev + (size_t)r * Ds * Ds, p.Vd_prev + (size_t)r * D * Ds, mx, sx, sc);
    }
    if (t >= p.H) return;
    double* mh = g.mh + (size_t)r * Dh;
    double* Sh = g.Sh + (size_t)r * Dh * Dh;
    dev_trig(g.tm, mx, sx, mh, Sh, g.Ch + (size_t)r * Ds * Dh);
    nz_noisy_cov(Ds, sx, z.var, sn);
    double* mz = z.mz + (size_t)r * Dh;
    double* Sz = z.Sz + (size_t)r * Dh * Dh;
    for (int k = tid; k < Dh; k += nt) mz[k] = trig_M_entry(g.tm, mx, sn, k);
    for (int e = tid; e < Dh * Dh; e += nt) Sz[e] = trig_S_entry(g.tm, mx, sn, e / Dh, e % Dh);
    __syncthreads();
    if (p.pol_kind == PILCO_POLICY_LINEAR) {
        dev_linear_action(Dh, U, p.W + (size_t)r * p.W_bs, p.b + (size_t)r * p.b_bs, mz, Sz,
                          p.Mp + (size_t)r * U, p.Sp + (size_t)r * U * U, p.Vp + (size_t)r * Dh * U, sc);
        ro_action_tail(p, r, mh, Sh, sc);
        tg_cross(g, r, sx, sc);
    }
}

__global__ void __launch_bounds__(128) nz_trig_kernel(NzBwdDev z) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    __shared__ double sn[TRIG_MAX * TRIG_MAX];
    const TbDev& g = z.g;
    const RbDev& p = g.p;
    const int r = blockIdx.x, Ds = g.tm.Ds, Dh = p.Ds, U = p.U, t = p.t;
    double* gm = p.gm + (size_t)r * Ds;
    double* gS = p.gS + (size_t)r * Ds * Ds;
    double* gmz = z.gmz + (size_t)r * Dh;
    double* gSz = z.gSz + (size_t)r * Dh * Dh;
    const double* mx = p.traj_m + ((size_t)r * (p.H + 1) + t) * Ds;
    const double* sx = p.traj_S + ((size_t)r * (p.H + 1) + t) * Ds * Ds;
    if (p.pol_kind == PILCO_POLICY_LINEAR)
        dev_linear_bwd(Dh, U, p.W + (size_t)r * p.W_bs, z.mz + (size_t)r * Dh, z.Sz + (size_t)r * Dh * Dh,
                       p.gMp + (size_t)r * U, p.gSp + (size_t)r * U * U, p.gVp + (size_t)r * Dh * U,
                       p.gW + (size_t)r * U * Dh, p.gb + (size_t)r * U, gmz, gSz, sc);
    dev_trig_bwd(g.tm, mx, sx, g.gmh + (size_t)r * Dh, g.gSh + (size_t)r * Dh * Dh, g.gCh + (size_t)r * Ds * Dh, gm, gS);
    nz_noisy_cov(Ds, sx, z.var, sn);
    dev_trig_bwd(g.tm, mx, sn, gmz, gSz, nullptr, gm, gS);
    for (int i = threadIdx.x; i < Dh; i += blockDim.x) gmz[i] = 0.0;            // ready for step t-1
    for (int e = threadIdx.x; e < Dh * Dh; e += blockDim.x) gSz[e] = 0.0;
    tg_trig_tail(g, r, gm, gS);
}

int nz_state_launch(const TgDev& g, const double* var, double* mz, double* Sz, cudaStream_t st) {
    NzDev z;
    z.g = g; z.mz = mz; z.Sz = Sz;
    for (int i = 0; i < MAXD; ++i) z.var[i] = var[i];
    launch_hi(nz_state_kernel, dim3(g.p.R), dim3(128), 0, st, z);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int nz_trig_launch(const TbDev& g, const double* var, const double* mz, const double* Sz, double* gmz, double* gSz,
                   cudaStream_t st) {
    NzBwdDev z;
    z.g = g; z.mz = mz; z.Sz = Sz; z.gmz = gmz; z.gSz = gSz;
    for (int i = 0; i < MAXD; ++i) z.var[i] = var[i];
    launch_hi(nz_trig_kernel, dim3(g.p.R), dim3(128), 0, st, z);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}
