// rollout_explore.cu -- the exploration objective of the original PILCO on the moment-matching rollout
// (pilco_rollout_explore_*): reward[r] = sum_t (E[r_t] + b sigma_t) (+ the MULT channel's term), with
//   sigma_t^2 = sum_k c_k^2 Var[r_k(x_t)] over the ADD-channel terms (CombinedRewards.compute_reward's rule, covariances
//   between terms ignored; state terms at (m_t, S_t), joint terms at step t's joint Gaussian), Var = r_2 - r_1^2 for an
//   exponential term (reward.m:52-56) and W^T S W for a linear one;  sigma_t = sqrt(sigma_t^2) above 1e-12 (reward.m:57),
//   else 0 with zero gradient.
// The kernels run off the serial chain, launched by the forward (rollout.cu) and the reverse sweep (rollout_bwd.cu) only
// with an active exploration, so the launches of a rollout without exploration are exactly those it always ran:
//   forward, after the reward launches:  ro_reward_var (t, r), ro_reward_joint_var (t, r; with a joint term), then
//            ro_reward_explore_sum in place of ro_reward_sum
//   reverse sweep with b != 0, after the reward-gradient precompute:  rb_reward_var (r, t) and rb_reward_joint_var (with
//            a joint term) add b c_k^2 / (2 sigma_t) dVar_k/d(m, S) to the ADD-channel slots that the per-step chain consumes
// A translation unit of its own, so that the existing kernels compile exactly as they do without it.
#include <cmath>

#include "rollout_bwd.cuh"
#include "small_kernels.cuh"

// sigma_t^2 below this is treated as 0 (reward.m:57)
#define EX_VAR_FLOOR 1e-12

// sigma_t^2 of the state terms, CTA = (step t, restart r): var[t R + r] = sum_k c_k^2 Var_k over the ADD-channel terms
__global__ void __launch_bounds__(128) ro_reward_var_kernel(RoDev p, double* var) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    __shared__ double vk;
    const int t = blockIdx.x, r = blockIdx.y, Ds = p.Ds;
    const double* mx = p.traj_m + ((size_t)r * (p.H + 1) + t) * Ds;
    const double* sx = p.traj_S + ((size_t)r * (p.H + 1) + t) * Ds * Ds;
    double v = 0.0;                                   // meaningful on thread 0, which writes vk
    for (int k = 0; k < p.n_rewards; ++k) {
        const pilco_reward_term& rt = p.rewards[k];
        if (rt.channel != PILCO_CHANNEL_ADD) continue;
        if (rt.kind == PILCO_REWARD_EXP) dev_exp_reward(Ds, rt.W, rt.t, mx, sx, &vk, sc);
        else dev_linear_reward(Ds, rt.W, mx, sx, &vk);           // an ADD-channel box term is rejected before launch
        if (threadIdx.x == 0) v = fma(rt.coef * rt.coef, vk, v);
    }
    if (threadIdx.x == 0) var[(size_t)t * p.R + r] = v;
}

// the joint state-action terms' share, CTA = (step t, restart r): p.rewards holds those terms only, p.mj / p.sj the joint
// Gaussians of step 0 (as ro_reward_joint); adds to what ro_reward_var wrote
__global__ void __launch_bounds__(128) ro_reward_joint_var_kernel(RoDev p, double* var) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    __shared__ double vk;
    const int t = blockIdx.x, r = blockIdx.y, D = p.Ds + p.U;
    const double* mj = p.mj + ((size_t)t * p.R + r) * D;
    const double* sj = p.sj + ((size_t)t * p.R + r) * D * D;
    __shared__ double v;                              // the running sum, on thread 0 (in a register it spills)
    if (threadIdx.x == 0) v = var[(size_t)t * p.R + r];
    for (int k = 0; k < p.n_rewards; ++k) {
        const pilco_reward_term& rt = p.rewards[k];
        if (rt.channel != PILCO_CHANNEL_ADD) continue;
        if (rt.kind == PILCO_REWARD_EXP_SA) dev_exp_reward(D, rt.W, rt.t, mj, sj, &vk, sc);
        else dev_linear_reward(D, rt.W, mj, sj, &vk);
        if (threadIdx.x == 0) v = fma(rt.coef * rt.coef, vk, v);
    }
    if (threadIdx.x == 0) var[(size_t)t * p.R + r] = v;
}

// reward[r] = sum_t (rew[t, r] + b sigma_t) in step order (+ mult_mu (1 - prod_t (1 - risk_t))); step_var [R,H] if set
__global__ void __launch_bounds__(128) ro_reward_explore_sum_kernel(RoDev p, double b, const double* var,
                                                                    double* step_var) {
    PDL_ENTRY();
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= p.R) return;
    double s = 0.0;
    for (int tt = 0; tt < p.H; ++tt) {
        const double v = var[(size_t)tt * p.R + r];
        const double sig = v > EX_VAR_FLOOR ? sqrt(v) : 0.0;
        s += p.rew[(size_t)tt * p.R + r] + b * sig;
        if (step_var) step_var[(size_t)r * p.H + tt] = v;
    }
    if (p.n_mult > 0) {
        double mult = 1.0;
        for (int tt = 0; tt < p.H; ++tt) mult *= 1.0 - p.risk[(size_t)tt * p.R + r];
        s += p.mult_mu * (1.0 - mult);
    }
    p.reward[r] = s;
}

// b c_k^2 / (2 sigma_t) dVar_k/d(m_t, S_t) of the state ADD terms into the ADD-channel slots rgm / rgS[t][0],
// CTA = (restart r, step t) as rb_reward
__global__ void __launch_bounds__(128) rb_reward_var_kernel(RbDev p, double b, const double* var) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    // w = b / (2 sigma_t) in shared memory and the pointers formed per term: so laid out, the kernel does not spill
    __shared__ double w;
    const int r = blockIdx.x, t = blockIdx.y, Ds = p.Ds;
    const double v = var[(size_t)t * p.R + r];
    if (!(v > EX_VAR_FLOOR)) return;
    if (threadIdx.x == 0) w = b / (2.0 * sqrt(v));
    __syncthreads();
    const size_t tr = (size_t)r * (p.H + 1) + t, o = ((size_t)t * 2) * p.R + r;
    for (int k = 0; k < p.n_rewards; ++k) {
        const pilco_reward_term& rt = p.rewards[k];
        if (rt.channel != PILCO_CHANNEL_ADD) continue;
        const double scale = w * rt.coef * rt.coef;
        const double* mx = p.traj_m + tr * Ds;
        const double* sx = p.traj_S + tr * Ds * Ds;
        double* gm = p.rgm + o * Ds;
        double* gS = p.rgS + o * Ds * Ds;
        if (rt.kind == PILCO_REWARD_EXP) {                         // Var = r_2 - r_1^2
            dev_exp_moment_bwd(Ds, rt.W, rt.t, mx, sx, 2.0, 1, scale, gm, gS, sc);
            dev_exp_moment_bwd(Ds, rt.W, rt.t, mx, sx, 1.0, 2, -scale, gm, gS, sc);
        } else {                                                   // Var = W^T S W
            for (int e = threadIdx.x; e < Ds * Ds; e += blockDim.x) gS[e] += scale * rt.W[e / Ds] * rt.W[e % Ds];
            __syncthreads();
        }
    }
}

// the same for the joint state-action terms at the forward's joint Gaussians, into jgm / jgS[t][0]
__global__ void __launch_bounds__(128) rb_reward_joint_var_kernel(RbDev p, double b, const double* var) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    const int r = blockIdx.x, t = blockIdx.y, D = p.Ds + p.U;
    const double v = var[(size_t)t * p.R + r];
    if (!(v > EX_VAR_FLOOR)) return;
    const double w = b / (2.0 * sqrt(v));
    const double* mj = p.mj0 + ((size_t)t * p.R + r) * D;
    const double* sj = p.sj0 + ((size_t)t * p.R + r) * D * D;
    double* gm = p.jgm + (((size_t)t * 2) * p.R + r) * D;
    double* gS = p.jgS + (((size_t)t * 2) * p.R + r) * D * D;
    for (int k = 0; k < p.n_rewards; ++k) {
        const pilco_reward_term& rt = p.rewards[k];
        if (rt.channel != PILCO_CHANNEL_ADD) continue;
        const double scale = w * rt.coef * rt.coef;
        if (rt.kind == PILCO_REWARD_EXP_SA) {
            dev_exp_moment_bwd(D, rt.W, rt.t, mj, sj, 2.0, 1, scale, gm, gS, sc);
            dev_exp_moment_bwd(D, rt.W, rt.t, mj, sj, 1.0, 2, -scale, gm, gS, sc);
        } else {
            for (int e = threadIdx.x; e < D * D; e += blockDim.x) gS[e] += scale * rt.W[e / D] * rt.W[e % D];
            __syncthreads();
        }
    }
}

int ex_reward_var_launch(const RoDev& ds, const RoDev* dj, double b, double* var, double* step_var, cudaStream_t st) {
    if (ds.H > 0) {
        launch_hi(ro_reward_var_kernel, dim3(ds.H, ds.R), dim3(128), 0, st, ds, var);
        CUDA_LAUNCH_CHECK();
        if (dj) {
            launch_hi(ro_reward_joint_var_kernel, dim3(dj->H, dj->R), dim3(128), 0, st, *dj, var);
            CUDA_LAUNCH_CHECK();
        }
    }
    launch_hi(ro_reward_explore_sum_kernel, dim3((ds.R + 127) / 128), dim3(128), 0, st, ds, b, (const double*)var, step_var);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int rb_reward_var_launch(const RbDev& ds, const RbDev* dj, double b, const double* var, cudaStream_t st) {
    launch_hi(rb_reward_var_kernel, dim3(ds.R, ds.H), dim3(128), 0, st, ds, b, var);
    CUDA_LAUNCH_CHECK();
    if (dj) {
        launch_hi(rb_reward_joint_var_kernel, dim3(dj->R, dj->H), dim3(128), 0, st, *dj, b, var);
        CUDA_LAUNCH_CHECK();
    }
    return PILCO_OK;
}
