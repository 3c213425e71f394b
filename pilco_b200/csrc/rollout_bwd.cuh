// rollout_bwd.cuh -- parameters of the reverse sweep's per-step kernels, shared by its driver (rollout_bwd.cu) and the
// kernels on phi (rollout_angles_bwd.cu), with measurement noise (rollout_noise.cu) and exploration (rollout_explore.cu).
#pragma once
#include "rollout.cuh"

struct MMTapeBwd;

static inline bool rb_has_joint(const pilco_rollout* ro) {
    for (int k = 0; k < ro->n_rewards && k < 8; ++k) if (reward_on_joint(ro->rewards[k].kind)) return true;
    return false;
}

struct RbDev {
    int R, H, Ds, U, t;
    int pol_kind, squash;
    const double* maxa;
    const double* W; long long W_bs;
    int n_rewards; pilco_reward_term rewards[8];
    const double* traj_m; const double* traj_S;
    const double* risk; double mult_mu;       // MULT channel: per-step risks risk[t*R + r] saved by the forward
    // forward slots of step t
    const double *sj, *Vd, *Mp, *Sp, *Vp, *Mu, *Su, *Cq, *Vu;
    // cotangent buffers [R, len]
    double *gm, *gS, *gMd, *gSd, *gVd, *gmj, *gsj, *gsjx, *gMp, *gSp, *gVp;
    double *gW, *gb;      // linear policy gradient accumulators [R,U,Ds], [R,U]
    double *rgm, *rgS;    // reward gradients of every step (rb_reward_kernel)
    double *jgm, *jgS;    // the joint state-action terms' gradients of every step, NULL without such terms
    const double *mj0, *sj0;  // forward joint Gaussians of step 0; step t is R D (R D D) doubles further on
    // taped dynamics VJP: task partials [R][ntask][MAXD + D*D] that rb_post sums into gmj / gsj itself (else NULL);
    // then the glue cotangent gsjx is formed in shared memory too (no rb_pre launch)
    const double* tpart; int tp_ntask;
    unsigned* cnt;
};

// rb_reward_kernel (state terms of ds, at dimension ds.Ds) and, when dj is non-NULL, rb_reward_joint_kernel (joint terms,
// at dimension dj->Ds + dj->U) (rollout_bwd.cu)
int rb_reward_launch(const RbDev& ds, const RbDev* dj, cudaStream_t st);
// the exploration gradient (rollout_explore.cu), once rb_reward_launch is enqueued and before the serial per-step
// chain: rb_reward_var with ds and, when dj is non-NULL, rb_reward_joint_var with dj, at sigma_t^2 var [H][R]
int rb_reward_var_launch(const RbDev& ds, const RbDev* dj, double b, const double* var, cudaStream_t st);

// parameters of the reverse per-step kernels on phi (rollout_angles_bwd.cu)
struct TbDev {
    RbDev p;                  // p.Ds = Dh; p.gm / p.gS: the raw state's cotangent [R, Ds], [R, Ds, Ds]
    TrigMap tm;
    const double *mh, *Sh, *Ch, *cx;  // forward slots of step t
    const double *cx_prev, *Vd_prev;  // step t-1 (NULL at t = 0)
    double *gVd, *gcx, *gmh, *gSh, *gCh;
};

#ifdef __CUDACC__
// the per-step trig stage once the trig VJP is in the state cotangent (gm, gS) of restart r: the state reward gradients
// of step t, then the symmetric part of gS0 (t = 0) or the seeds of step t-1.  The tail of tg_trig_kernel
// (rollout_angles_bwd.cu), which keeps its own copy: calling this from it changes that kernel's register allocation.
__device__ __forceinline__ void tg_trig_tail(const TbDev& g, int r, double* gm, double* gS) {
    const RbDev& p = g.p;
    const int Ds = g.tm.Ds, Dh = p.Ds, D = Dh + p.U, t = p.t;
    const int tid = threadIdx.x, nt = blockDim.x;
    double wmult = p.mult_mu;
    if (wmult != 0.0)
        for (int tt = 0; tt < p.H; ++tt) if (tt != t) wmult *= 1.0 - p.risk[(size_t)tt * p.R + r];
    const double* ra_m = p.rgm + (((size_t)t * 2) * p.R + r) * Ds;
    const double* ra_S = p.rgS + (((size_t)t * 2) * p.R + r) * Ds * Ds;
    const double* rm_m = ra_m + (size_t)p.R * Ds;
    const double* rm_S = ra_S + (size_t)p.R * Ds * Ds;
    for (int i = tid; i < Ds; i += nt) gm[i] += ra_m[i] + wmult * rm_m[i];
    for (int e = tid; e < Ds * Ds; e += nt) gS[e] += ra_S[e] + wmult * rm_S[e];
    __syncthreads();
    if (t == 0) {              // gS0: the symmetric part (S0 is symmetric; the glue's gQ C^T terms are not)
        for (int e = tid; e < Ds * Ds; e += nt) {
            const int i = e / Ds, j = e % Ds;
            if (i < j) { const double v = 0.5 * (gS[e] + gS[j * Ds + i]); gS[e] = v; gS[j * Ds + i] = v; }
        }
        return;
    }
    // seeds of step t-1: gV = cx^T (gS + gS^T) [D, Ds],  gcx = (gS + gS^T) V_d^T [Ds, D]
    const double* cx = g.cx_prev + (size_t)r * Ds * D;
    const double* Vd = g.Vd_prev + (size_t)r * D * Ds;
    for (int e = tid; e < D * Ds; e += nt) {
        const int k = e / Ds, j = e % Ds;
        double v = 0.0;
        for (int i = 0; i < Ds; ++i) v = fma(cx[i * D + k], gS[i * Ds + j] + gS[j * Ds + i], v);
        g.gVd[(size_t)r * D * Ds + e] = v;
    }
    for (int e = tid; e < Ds * D; e += nt) {
        const int i = e / D, k = e % D;
        double v = 0.0;
        for (int j = 0; j < Ds; ++j) v = fma(gS[i * Ds + j] + gS[j * Ds + i], Vd[k * Ds + j], v);
        g.gcx[(size_t)r * Ds * D + e] = v;
    }
}
#endif

// the post stage of step g.p.t on phi (rollout_angles_bwd.cu): with a tape (tb) tg_dyn_finish, the tape-driven dynamics
// VJP whose last CTA of a restart runs tg_post, else tg_post alone after the recomputing dynamics VJP
int tg_post_launch(const TbDev& g, const MMTapeBwd* tb, cudaStream_t st);
// the trig stage of step g.p.t (rollout_angles_bwd.cu): trig VJP, state reward gradients, seeds of step t-1
int tg_trig_launch(const TbDev& g, cudaStream_t st);
// the per-step trig stage of the noisy reverse sweep (in place of tg_trig; rollout_noise.cu): the linear-policy VJP at
// the noisy moments (mz, Sz) into (gmz, gSz), both trig VJPs into the state cotangent, then tg_trig's reward gradients
// and seeds of step t-1; (gmz, gSz) are left zero for the next step.  var: the noise variances [MAXD]
int nz_trig_launch(const TbDev& g, const double* var, const double* mz, const double* Sz, double* gmz, double* gSz,
                   cudaStream_t st);
int rbf_factor_bwd_launch(cudaStream_t st, int R, int bf, int Ds, int U, const double* X, long long X_bs,
                          const double* ell, long long ell_bs, const double* sf2, long long sf2_bs,
                          const double* beta, long long beta_bs, const double* gy,
                          double* gX, double* gY, double* gell);
