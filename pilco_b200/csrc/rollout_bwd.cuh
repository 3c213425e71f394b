// rollout_bwd.cuh -- parameters of the reverse sweep's per-step kernels, shared by rollout_bwd.cu and the reverse sweep
// with angular state dimensions (rollout_angles_bwd.cu).
#pragma once
#include "rollout.cuh"

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

int rb_reward_launch(const RbDev& ds, const RbDev* dj, cudaStream_t st);
// Optional hook of the reverse sweep (pilco_rollout_explore_backward): run once the reward-gradient precompute
// (rb_reward, rb_reward_joint) is enqueued and before the serial per-step chain, with the state terms' parameters ds
// (state dimension ds.Ds) and, when a joint state-action term is present, the joint terms' dj, else NULL.
typedef int (*RbRewardHook)(const RbDev& ds, const RbDev* dj, cudaStream_t st, const void* ctx);
// pilco_rollout_backward with the hook above (rollout_bwd.cu); hook == NULL is that call
int rb_backward_impl(const pilco_rollout* ro, const pilco_rollout_grad* g, RbRewardHook hook, const void* ctx,
                     cudaStream_t st);
// pilco_rollout_angles_backward (ang may be NULL) with the hook above (rollout_angles_bwd.cu)
int rb_backward_run(const pilco_rollout* ro, const pilco_angles* ang, const pilco_rollout_grad* g, RbRewardHook hook,
                    const void* ctx, cudaStream_t st);
int rbf_factor_bwd_launch(cudaStream_t st, int R, int bf, int Ds, int U, const double* X, long long X_bs,
                          const double* ell, long long ell_bs, const double* sf2, long long sf2_bs,
                          const double* beta, long long beta_bs, const double* gy,
                          double* gX, double* gY, double* gell);
