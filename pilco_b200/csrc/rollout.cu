// rollout.cu -- H-step moment-matching cascade (forward), one batch of R independent rollouts.
// Replaces PILCO.predict / PILCO.propagate (pilco/models/pilco.py:118-153; pred.m, propagate.m).
//
// Launch sequence per step t (all on one stream, graph-capturable, no host sync):
//   ro_state<t>   grid R : [t>0: finish dynamics MM of step t-1 + next-state glue] -> traj[t];
//                          linear policy + squash + joint Gaussian
//   (RBF policy)  mm_setup/mm_tile on the policy GP, then ro_policy<t>: finish + squash + joint
//   mm_setup / mm_tile on the dynamics GP with the joint Gaussian of step t
// and a final ro_state<H> that closes the last step.  The expected rewards depend on the trajectory only, so they are
// NOT on this chain (an LU factorisation per step and restart would sit on the serial path of every step): one
// ro_reward launch over all (t, r) after the last step, then ro_reward_sum adds them in step order (same summation
// order, hence the same bits, as a running sum).  Terms on the joint state-action Gaussian (PILCO_REWARD_*_SA) read
// the per-step joints the cascade keeps in the workspace for the reverse sweep: ro_reward_joint, launched between the two
// only when such a term is present, adds them to each step's reward and risk (state terms first, then joint terms, each in
// term order).  ro_reward sees the state terms only, so a rollout without joint terms runs exactly the kernels it always ran.
#include <cmath>

#include "rollout.cuh"
#include "mm_tape.cuh"
#include "small_kernels.cuh"
#include "rollout_step.cuh"

__global__ void __launch_bounds__(128) ro_state_kernel(RoDev p) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    const int r = blockIdx.x, t = p.t, Ds = p.Ds, U = p.U, D = Ds + U;
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
        const double* mxp = mx - Ds;
        const double* sxp = sx - Ds * Ds;
        dev_glue(Ds, U, mxp, sxp, p.sj_prev + (size_t)r * D * D,
                 p.Md_prev + (size_t)r * Ds, p.Sd_prev + (size_t)r * Ds * Ds, p.Vd_prev + (size_t)r * D * Ds,
                 mx, sx, sc);
    }
    if (t >= p.H) return;
    if (p.pol_kind == PILCO_POLICY_LINEAR) {
        dev_linear_action(Ds, U, p.W + (size_t)r * p.W_bs, p.b + (size_t)r * p.b_bs, mx, sx,
                          p.Mp + (size_t)r * U, p.Sp + (size_t)r * U * U, p.Vp + (size_t)r * Ds * U, sc);
        ro_action_tail(p, r, mx, sx, sc);
    }
}

__global__ void __launch_bounds__(128) ro_policy_kernel(RoDev p) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    const int r = blockIdx.x, t = p.t, Ds = p.Ds;
    mm_finish_device(p.pol, r);
    __syncthreads();
    const double* mx = p.traj_m + ((size_t)r * (p.H + 1) + t) * Ds;
    const double* sx = p.traj_S + ((size_t)r * (p.H + 1) + t) * Ds * Ds;
    ro_action_tail(p, r, mx, sx, sc);
}

// expected reward at the pre-step state of every step (pilco.py:130-134), CTA = (step t, restart r)
__global__ void __launch_bounds__(128) ro_reward_kernel(RoDev p) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    const int t = blockIdx.x, r = blockIdx.y, Ds = p.Ds;
    const double* mx = p.traj_m + ((size_t)r * (p.H + 1) + t) * Ds;
    const double* sx = p.traj_S + ((size_t)r * (p.H + 1) + t) * Ds * Ds;
    double rew = 0.0, risk = 0.0;
    for (int k = 0; k < p.n_rewards; ++k) {
        const pilco_reward_term& rt = p.rewards[k];
        const double mu = dev_reward_value(Ds, rt, mx, sx, sc);
        if (rt.channel == PILCO_CHANNEL_MULT) risk = fma(rt.coef, mu, risk);
        else rew = fma(rt.coef, mu, rew);
    }
    if (threadIdx.x == 0) {
        p.rew[(size_t)t * p.R + r] = rew;
        if (p.step_reward) p.step_reward[(size_t)r * p.H + t] = rew;
        if (p.n_mult > 0) {
            p.risk[(size_t)t * p.R + r] = risk;
            if (p.step_risk) p.step_risk[(size_t)r * p.H + t] = risk;
        }
    }
}

// the joint state-action terms of every step, CTA = (step t, restart r): p.rewards holds those terms only and p.mj, p.sj
// the joint Gaussians of step 0 (step t is R D, R D D doubles further on): what the dynamics moment match of step t received
__global__ void __launch_bounds__(128) ro_reward_joint_kernel(RoDev p) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    const int t = blockIdx.x, r = blockIdx.y, D = p.Ds + p.U;
    const double* mj = p.mj + ((size_t)t * p.R + r) * D;
    const double* sj = p.sj + ((size_t)t * p.R + r) * D * D;
    const size_t o = (size_t)t * p.R + r;
    double rew = p.rew[o], risk = p.n_mult > 0 ? p.risk[o] : 0.0;
    for (int k = 0; k < p.n_rewards; ++k) {
        const pilco_reward_term& rt = p.rewards[k];
        const double mu = dev_joint_reward_value(D, rt, mj, sj, sc);
        if (rt.channel == PILCO_CHANNEL_MULT) risk = fma(rt.coef, mu, risk);
        else rew = fma(rt.coef, mu, rew);
    }
    if (threadIdx.x == 0) {
        p.rew[o] = rew;
        if (p.step_reward) p.step_reward[(size_t)r * p.H + t] = rew;
        if (p.n_mult > 0) {
            p.risk[o] = risk;
            if (p.step_risk) p.step_risk[(size_t)r * p.H + t] = risk;
        }
    }
}

// reward[r] = sum_t rew[t, r] in step order  (+ SafePILCO.predict, safe_pilco.py:49: mu (1 - prod_t (1 - risk_t)))
__global__ void __launch_bounds__(128) ro_reward_sum_kernel(RoDev p) {
    PDL_ENTRY();
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= p.R) return;
    double s = 0.0;
    for (int tt = 0; tt < p.H; ++tt) s += p.rew[(size_t)tt * p.R + r];
    if (p.n_mult > 0) {
        double mult = 1.0;
        for (int tt = 0; tt < p.H; ++tt) mult *= 1.0 - p.risk[(size_t)tt * p.R + r];
        s += p.mult_mu * (1.0 - mult);
    }
    p.reward[r] = s;
}

// ---------------------------------------------------------------------------------------------
// Angular state dimensions (pilco_rollout_angles_forward).  The state x [Ds] stays raw; the policy and the dynamics GP
// see phi(x) [Dh] (trig_math.cuh).  Per step t:
//   tg_state<t>   grid R : [t>0: finish dynamics MM of step t-1 + glue with cx_{t-1}] -> traj[t]; phi moments (m^, S^, C^);
//                          linear policy on (m^, S^) + squash + joint [phi, u] + cx_t
//   (RBF policy)  mm_setup/mm_tile on the policy GP at (m^, S^), then tg_policy<t>: finish + squash + joint + cx_t
//   mm_setup / mm_tile on the dynamics GP with the joint Gaussian of step t (D = Dh + U)
// cx_t = cov(x_t, [phi(x_t), u_t]) = S_x C^ [I, V_u] [Ds, Dh + U] takes the place of the first Ds rows of the joint
// covariance in the glue: S' = S_x + S_d + cx V_d + (cx V_d)^T.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) tg_state_kernel(TgDev g) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
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
        // dev_glue reads the first Ds rows of a [., Ds + U'] matrix: cx [Ds, Dh + U] with U' = Dh + U - Ds
        const int D = Dh + U;
        dev_glue(Ds, D - Ds, mx - Ds, sx - Ds * Ds, g.cx_prev + (size_t)r * Ds * D,
                 p.Md_prev + (size_t)r * Ds, p.Sd_prev + (size_t)r * Ds * Ds, p.Vd_prev + (size_t)r * D * Ds, mx, sx, sc);
    }
    if (t >= p.H) return;
    double* mh = g.mh + (size_t)r * Dh;
    double* Sh = g.Sh + (size_t)r * Dh * Dh;
    dev_trig(g.tm, mx, sx, mh, Sh, g.Ch + (size_t)r * Ds * Dh);
    if (p.pol_kind == PILCO_POLICY_LINEAR) {
        dev_linear_action(Dh, U, p.W + (size_t)r * p.W_bs, p.b + (size_t)r * p.b_bs, mh, Sh,
                          p.Mp + (size_t)r * U, p.Sp + (size_t)r * U * U, p.Vp + (size_t)r * Dh * U, sc);
        ro_action_tail(p, r, mh, Sh, sc);
        tg_cross(g, r, sx, sc);
    }
}

__global__ void __launch_bounds__(128) tg_policy_kernel(TgDev g) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    const RoDev& p = g.p;
    const int r = blockIdx.x, t = p.t, Ds = g.tm.Ds, Dh = p.Ds;
    mm_finish_device(p.pol, r);
    __syncthreads();
    const double* sx = p.traj_S + ((size_t)r * (p.H + 1) + t) * Ds * Ds;
    ro_action_tail(p, r, g.mh + (size_t)r * Dh, g.Sh + (size_t)r * Dh * Dh, sc);
    tg_cross(g, r, sx, sc);
}

// validation of a rollout whose dynamics GP predicts E outputs (the state dimension): E = pol.Ds without angles
static int ro_check_as(const pilco_rollout* ro, int E) {
    if (ro->R < 1 || ro->H < 0) return PILCO_ERR_DIM;
    int rc = mm_check_model(&ro->dyn);
    if (rc) return rc;
    const int Ds = ro->pol.Ds, U = ro->pol.U;
    if (Ds < 1 || U < 1 || Ds + U != ro->dyn.D || ro->dyn.E != E) return PILCO_ERR_DIM;
    if (ro->pol.squash && !ro->pol.max_action) return PILCO_ERR_NULL;
    if (ro->pol.kind == PILCO_POLICY_LINEAR) { if (!ro->pol.W || !ro->pol.b) return PILCO_ERR_NULL; }
    else if (ro->pol.kind == PILCO_POLICY_RBF) {
        rc = mm_check_model(&ro->pol.rbf);
        if (rc) return rc;
        if (ro->pol.rbf.D != Ds || ro->pol.rbf.E != U || ro->pol.rbf.mode != 1) return PILCO_ERR_DIM;
    } else return PILCO_ERR_UNSUPPORTED;
    if (ro->n_rewards < 1 || ro->n_rewards > 8) return PILCO_ERR_DIM;
    for (int k = 0; k < ro->n_rewards; ++k) {
        if (!ro->rewards[k].W) return PILCO_ERR_NULL;
        const int kind = ro->rewards[k].kind, ch = ro->rewards[k].channel;
        if (reward_needs_t(kind) && !ro->rewards[k].t) return PILCO_ERR_NULL;
        if (!reward_kind_known(kind)) return PILCO_ERR_UNSUPPORTED;
        if (ch != PILCO_CHANNEL_ADD && ch != PILCO_CHANNEL_MULT) return PILCO_ERR_UNSUPPORTED;
    }
    if (!ro->m0 || !ro->S0 || !ro->traj_m || !ro->traj_S || !ro->reward || !ro->ws) return PILCO_ERR_NULL;
    return PILCO_OK;
}

int ro_validate(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex, const pilco_obs_noise* nz,
                bool backward, RoOpt* o, const pilco_policy_schedule* sch) {
    *o = RoOpt{};
    if (!ro) return PILCO_ERR_NULL;
    const int A = ang ? ang->A : 0, Ds = ro->dyn.E;
    if (A != 0) {                                     // the angles before the rest of the description
        if (trig_map_make(Ds, A, ang->dims, &o->tm) || Ds + A + ro->pol.U > MAXD) return PILCO_ERR_DIM;
        if (ro->pol.Ds != Ds + A) return PILCO_ERR_DIM;
    }
    int rc = ro_check_as(ro, A != 0 ? Ds : ro->pol.Ds);
    if (rc) return rc;
    o->explore = ex_active(ex);
    if (o->explore) {
        if (!std::isfinite(ex->b)) return PILCO_ERR_DIM;
        for (int k = 0; k < ro->n_rewards; ++k)       // no variance closed form for a box term
            if (ro->rewards[k].channel == PILCO_CHANNEL_ADD && ro->rewards[k].kind == PILCO_REWARD_BOX)
                return PILCO_ERR_UNSUPPORTED;
        o->b = ex->b; o->step_var = ex->step_var;
    }
    o->noise = nz != nullptr;
    for (int i = 0; i < MAXD; ++i) {                  // Ds <= PILCO_MAX_D - 1 once the description has passed
        o->nzvar[i] = nz && i < Ds ? nz->var[i] : 0.0;
        if (!std::isfinite(o->nzvar[i]) || o->nzvar[i] < 0.0) return PILCO_ERR_DIM;
    }
    o->phi = ro_on_phi(ang, nz);
    if (o->phi && A == 0) trig_map_make(Ds, 0, nullptr, &o->tm);
    if (sch && (sch->W_ts < 0 || sch->b_ts < 0)) return PILCO_ERR_DIM;
    if (sch_active(sch) && ro->pol.kind != PILCO_POLICY_LINEAR) return PILCO_ERR_UNSUPPORTED;
    if ((!backward || o->explore || o->noise) && ro->ws_bytes < ro_ws_layout(ro, ang, ex, nz).total * sizeof(double))
        return PILCO_ERR_WORKSPACE;
    if (backward) return PILCO_OK;
    if (((uintptr_t)ro->ws) & 15) return PILCO_ERR_ALIGN;
    if (ro->tape) {
        const size_t need = pilco_rollout_tape_bytes(ro);
        if (need == 0 && ro->H > 0) return PILCO_ERR_UNSUPPORTED;
        if (ro->tape_bytes < need) return PILCO_ERR_WORKSPACE;
        if (((uintptr_t)ro->tape) & 15) return PILCO_ERR_ALIGN;
    }
    return PILCO_OK;
}

// The forward of every call (ang, ex, nz, sch may be NULL).  Per step the state kernel is ro_state, tg_state on phi or
// nz_state with noise, and the policy kernel ro_policy or tg_policy (on phi); the policy GP reads x_t, phi's moments or
// the noisy ones.  The state terms read the raw trajectory, the joint terms [phi, u]: ro_reward_joint's D = Dh + U.
// Every state kernel reads the linear policy through its launch's W and b, so a schedule advances them by a step's
// strides before each launch and no kernel changes.
static int ro_forward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                      const pilco_obs_noise* nz, const pilco_policy_schedule* sch, cudaStream_t st) {
    RoOpt o;
    int rc = ro_validate(ro, ang, ex, nz, false, &o, sch);
    if (rc) return rc;
    const RoWs L = ro_ws_layout(ro, ang, ex, nz);
    double* ws = (double*)ro->ws;
    const int R = ro->R, H = ro->H, Ds = ro->dyn.E, Dh = ro->pol.Ds, U = ro->pol.U, D = Dh + U;
    const size_t RR = (size_t)R;

    TgDev g;
    g.tm = o.tm;
    RoDev& d = g.p;
    d.R = R; d.H = H; d.Ds = Dh; d.U = U;
    d.pol_kind = ro->pol.kind; d.squash = ro->pol.squash; d.maxa = ro->pol.max_action;
    d.W = ro->pol.W; d.W_bs = ro->pol.W_bs; d.b = ro->pol.b; d.b_bs = ro->pol.b_bs;
    pilco_reward_term joint_terms[8];
    const int n_joint = ro_split_rewards(ro, &d.n_rewards, d.rewards, joint_terms);
    d.m0 = ro->m0; d.m0_bs = ro->m0_bs; d.S0 = ro->S0; d.S0_bs = ro->S0_bs;
    d.traj_m = ro->traj_m; d.traj_S = ro->traj_S; d.reward = ro->reward; d.step_reward = ro->step_reward;
    d.risk = ws + L.risk; d.rew = ws + L.rew; d.step_risk = ro->step_risk; d.mult_mu = ro->mult_mu; d.n_mult = ro_count_mult(ro);

    auto slot = [&](size_t base, size_t len, int t) { return ws + base + (size_t)t * RR * len; };
    const MMTapeL TL = ro->tape ? mm_tape_layout(ro->dyn.n, ro->dyn.D, ro->dyn.E, R) : MMTapeL();
    auto dyn_params = [&](int t) {                   // taped: the tile pass writes slot (t, :) of the rollout's tape
        return mm_params(&ro->dyn, R, slot(L.mj, D, t), D, slot(L.sj, (size_t)D * D, t), (long long)D * D,
                         slot(L.Md, Ds, t), slot(L.Sd, (size_t)Ds * Ds, t), slot(L.Vd, (size_t)D * Ds, t), ro->info,
                         ws + L.dynws, ro->tape ? (double*)ro->tape + (size_t)t * RR * TL.per_r : nullptr, TL);
    };
    const size_t pm = o.noise ? L.mz : L.mh, pS = o.noise ? L.Sz : L.Sh;
    auto pol_params = [&](int t) {
        return o.phi ? mm_params(&ro->pol.rbf, R, slot(pm, Dh, t), Dh, slot(pS, (size_t)Dh * Dh, t), (long long)Dh * Dh,
                                 slot(L.Mp, U, t), slot(L.Sp, (size_t)U * U, t), slot(L.Vp, (size_t)Dh * U, t), ro->info,
                                 ws + L.polws)
                     : mm_params(&ro->pol.rbf, R, ro->traj_m + (size_t)t * Ds, (long long)(H + 1) * Ds,
                                 ro->traj_S + (size_t)t * Ds * Ds, (long long)(H + 1) * Ds * Ds, slot(L.Mp, U, t),
                                 slot(L.Sp, (size_t)U * U, t), slot(L.Vp, (size_t)Dh * U, t), ro->info, ws + L.polws);
    };

    if (ro->info) cudaMemsetAsync(ro->info, 0, sizeof(int) * RR, st);
    const long long W_ts = sch_active(sch) ? sch->W_ts : 0, b_ts = sch_active(sch) ? sch->b_ts : 0;
    for (int t = 0; t <= H; ++t) {
        d.t = t;
        if (W_ts || b_ts) { d.W = ro->pol.W + (t < H ? t : 0) * W_ts; d.b = ro->pol.b + (t < H ? t : 0) * b_ts; }
        const int tc = t < H ? t : H - 1 < 0 ? 0 : H - 1;      // slot used for "current" pointers (unused at t==H)
        d.mj = slot(L.mj, D, tc); d.sj = slot(L.sj, (size_t)D * D, tc);
        d.Mp = slot(L.Mp, U, tc); d.Sp = slot(L.Sp, (size_t)U * U, tc); d.Vp = slot(L.Vp, (size_t)Dh * U, tc);
        d.Mu = slot(L.Mu, U, tc); d.Su = slot(L.Su, (size_t)U * U, tc); d.Cq = slot(L.Cq, (size_t)U * U, tc);
        d.Vu = slot(L.Vu, (size_t)Dh * U, tc);
        g.mh = slot(L.mh, Dh, tc); g.Sh = slot(L.Sh, (size_t)Dh * Dh, tc); g.Ch = slot(L.Ch, (size_t)Ds * Dh, tc);
        g.cx = slot(L.cx, (size_t)Ds * D, tc);
        if (t > 0) {
            d.mj_prev = slot(L.mj, D, t - 1); d.sj_prev = slot(L.sj, (size_t)D * D, t - 1);
            d.Md_prev = slot(L.Md, Ds, t - 1); d.Sd_prev = slot(L.Sd, (size_t)Ds * Ds, t - 1);
            d.Vd_prev = slot(L.Vd, (size_t)D * Ds, t - 1);
            g.cx_prev = slot(L.cx, (size_t)Ds * D, t - 1);
            d.dyn_prev = dyn_params(t - 1);
        } else {
            d.mj_prev = d.sj_prev = d.Md_prev = d.Sd_prev = d.Vd_prev = nullptr;
            g.cx_prev = nullptr;
            d.dyn_prev = dyn_params(0);
        }
        if (ro->pol.kind == PILCO_POLICY_RBF && t < H) d.pol = pol_params(t); else d.pol = d.dyn_prev;
        if (o.noise) {
            rc = nz_state_launch(g, o.nzvar, slot(L.mz, Dh, tc), slot(L.Sz, (size_t)Dh * Dh, tc), st);
            if (rc) return rc;
        } else {
            if (o.phi) launch_hi(tg_state_kernel, dim3(R), dim3(128), 0, st, g);
            else launch_hi(ro_state_kernel, dim3(R), dim3(128), 0, st, d);
            CUDA_LAUNCH_CHECK();
        }
        if (t == H) break;
        if (ro->pol.kind == PILCO_POLICY_RBF) {
            rc = mm_forward_launch(d.pol, st, false);
            if (rc) return rc;
            if (o.phi) launch_hi(tg_policy_kernel, dim3(R), dim3(128), 0, st, g);
            else launch_hi(ro_policy_kernel, dim3(R), dim3(128), 0, st, d);
            CUDA_LAUNCH_CHECK();
        }
        rc = mm_forward_launch(dyn_params(t), st, false);
        if (rc) return rc;
    }
    RoDev dr = d;
    dr.Ds = Ds;
    if (H > 0) {
        launch_hi(ro_reward_kernel, dim3(H, R), dim3(128), 0, st, dr);
        CUDA_LAUNCH_CHECK();
    }
    RoDev dj = d;
    dj.n_rewards = n_joint;
    for (int k = 0; k < 8; ++k) dj.rewards[k] = joint_terms[k];
    dj.mj = slot(L.mj, D, 0); dj.sj = slot(L.sj, (size_t)D * D, 0);
    if (H > 0 && n_joint > 0) {
        launch_hi(ro_reward_joint_kernel, dim3(H, R), dim3(128), 0, st, dj);
        CUDA_LAUNCH_CHECK();
    }
    if (o.explore) return ex_reward_var_launch(dr, n_joint > 0 ? &dj : nullptr, o.b, ws + L.var, o.step_var, st);
    launch_hi(ro_reward_sum_kernel, dim3((R + 127) / 128), dim3(128), 0, st, dr);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

// the size of the forward workspace: 0 for a description without a batch or with H < 0
static size_t ro_ws_bytes(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                          const pilco_obs_noise* nz, const pilco_policy_schedule* sch = nullptr) {
    if (!ro || ro->R < 1 || ro->H < 0 || (sch && (sch->W_ts < 0 || sch->b_ts < 0))) return 0;
    return ro_ws_layout(ro, ang, ex, nz).total * sizeof(double);
}

extern "C" {

size_t pilco_rollout_tape_bytes(const pilco_rollout* ro) {
    if (!ro || ro->R < 1 || ro->H < 0) return 0;
    if (!mm_tape_supported(ro->dyn.n, ro->dyn.D) || ro->dyn.D < 1 || ro->dyn.D > MAXD || ro->dyn.E < 1 || ro->dyn.E > MAXE) return 0;
    return mm_tape_layout(ro->dyn.n, ro->dyn.D, ro->dyn.E, ro->R).per_r * (size_t)ro->R * (size_t)ro->H * sizeof(double);
}

size_t pilco_rollout_angles_tape_bytes(const pilco_rollout* ro, const pilco_angles* ang) {
    (void)ang;                                        // the tape depends on the dynamics GP's shape only
    return pilco_rollout_tape_bytes(ro);
}

size_t pilco_rollout_workspace_bytes(const pilco_rollout* ro) { return ro_ws_bytes(ro, nullptr, nullptr, nullptr); }

size_t pilco_rollout_angles_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang) {
    return ro_ws_bytes(ro, ang, nullptr, nullptr);
}

size_t pilco_rollout_explore_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang,
                                             const pilco_exploration* ex) {
    return ro_ws_bytes(ro, ang, ex, nullptr);
}

size_t pilco_rollout_noisy_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                           const pilco_obs_noise* nz) {
    return ro_ws_bytes(ro, ang, ex, nz);
}

int pilco_rollout_forward(const pilco_rollout* ro, pilco_stream_t stream) {
    return ro_forward(ro, nullptr, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

int pilco_rollout_angles_forward(const pilco_rollout* ro, const pilco_angles* ang, pilco_stream_t stream) {
    return ro_forward(ro, ang, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}

int pilco_rollout_explore_forward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                  pilco_stream_t stream) {
    return ro_forward(ro, ang, ex, nullptr, nullptr, (cudaStream_t)stream);
}

int pilco_rollout_noisy_forward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                const pilco_obs_noise* nz, pilco_stream_t stream) {
    return ro_forward(ro, ang, ex, nz, nullptr, (cudaStream_t)stream);
}

size_t pilco_rollout_scheduled_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang,
                                               const pilco_exploration* ex, const pilco_obs_noise* nz,
                                               const pilco_policy_schedule* sch) {
    return ro_ws_bytes(ro, ang, ex, nz, sch);
}

int pilco_rollout_scheduled_forward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                    const pilco_obs_noise* nz, const pilco_policy_schedule* sch, pilco_stream_t stream) {
    return ro_forward(ro, ang, ex, nz, sch, (cudaStream_t)stream);
}

}  // extern "C"
