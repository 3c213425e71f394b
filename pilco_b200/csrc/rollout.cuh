// rollout.cuh -- workspace layout, validation and kernel parameters of the H-step cascade, shared by its forward
// (rollout.cu) and reverse sweep (rollout_bwd.cu) and the kernels of its options in their own translation units.
#pragma once
#include "mm_kernels.cuh"

#include "trig_math.cuh"

// The cascade runs on the features phi(x) of the state (trig_math.cuh) with angular state dimensions or measurement
// noise: with noise and no angles phi is the identity.  Without either the policy and the dynamics see x itself.
static inline bool ro_on_phi(const pilco_angles* ang, const pilco_obs_noise* nz) { return nz || (ang && ang->A != 0); }
// sigma_t^2 is computed (and its slot kept) when b != 0 or step_var is set
static inline bool ex_active(const pilco_exploration* ex) { return ex && (ex->b != 0.0 || ex->step_var); }

struct RoWs {                 // offsets in doubles into pilco_rollout.ws; per step [H][R][len] unless noted
    size_t mj, sj, Md, Sd, Vd, Mp, Sp, Vp, Mu, Su, Cq, Vu, risk, rew, mh, Sh, Ch, cx, dynws, polws, mz, Sz, var, total;
};

// The forward workspace.  Dh = pol.Ds is the policy's input dimension and E the dynamics GP's output count: dyn.E on
// phi, pol.Ds without.  A slot whose feature is off has length 0.
static inline RoWs ro_ws_layout(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                const pilco_obs_noise* nz) {
    const bool phi = ro_on_phi(ang, nz);
    const size_t R = ro->R, H = ro->H;
    const size_t Dh = ro->pol.Ds, U = ro->pol.U, D = Dh + U, E = phi ? (size_t)ro->dyn.E : Dh;
    const size_t F = phi ? 1 : 0, N = nz ? 1 : 0;
    RoWs L; size_t o = 0;
    auto take = [&](size_t len) { size_t at = o; o += (H * R * len + 1) & ~(size_t)1; return at; };
    L.mj = take(D); L.sj = take(D * D);
    L.Md = take(E); L.Sd = take(E * E); L.Vd = take(D * E);
    L.Mp = take(U); L.Sp = take(U * U); L.Vp = take(Dh * U);
    L.Mu = take(U); L.Su = take(U * U); L.Cq = take(U * U); L.Vu = take(Dh * U);
    L.risk = take(1);                       // per-step risk of the MULT reward channel, [H][R]
    L.rew = take(1);                        // per-step additive reward, [H][R] (summed in step order by ro_reward_sum_kernel)
    // on phi: its moments (m^, S^, C^) and cx = cov(x, [phi, u]) [E, Dh + U]
    L.mh = take(F * Dh); L.Sh = take(F * Dh * Dh); L.Ch = take(F * E * Dh); L.cx = take(F * E * D);
    L.dynws = o; o += pilco_mm_workspace_bytes(ro->dyn.n, ro->dyn.D, ro->dyn.E, ro->R) / 8;
    L.polws = o;
    if (ro->pol.kind == PILCO_POLICY_RBF)
        o += pilco_mm_workspace_bytes(ro->pol.rbf.n, ro->pol.rbf.D, ro->pol.rbf.E, ro->R) / 8;
    L.mz = take(N * Dh); L.Sz = take(N * Dh * Dh);     // measurement noise: phi's moments at N(m, S + diag(var))
    L.var = take(ex_active(ex) ? 1 : 0);               // exploration: sigma_t^2, [H][R]
    L.total = o;
    return L;
}

// what one validated call runs: ro_validate fills it
struct RoOpt {
    TrigMap tm;               // phi (the identity map of dyn.E dimensions with noise and no angles); meaningful on phi
    bool phi;                 // ro_on_phi
    bool noise;               // measurement noise at the policy's input, variances nzvar (0 from dyn.E on)
    double nzvar[MAXD];
    bool explore;             // ex_active
    double b; double* step_var;
};

// Validation of a call of the cascade (ang, ex, nz may be NULL) before anything is enqueued: the description, the
// angles, the exploration terms, the noise variances, then ro->ws's size (and for the forward its alignment and the
// tape).  The reverse sweep without exploration and noise does not check ro->ws.  A policy schedule (sch, may be NULL)
// is checked after the noise and before the workspace.
int ro_validate(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex, const pilco_obs_noise* nz,
                bool backward, RoOpt* o, const pilco_policy_schedule* sch = nullptr);

// a schedule that moves the policy's parameters with the step (pilco_rollout_scheduled_*); inactive: the stationary call
static inline bool sch_active(const pilco_policy_schedule* sch) { return sch && (sch->W_ts != 0 || sch->b_ts != 0); }

// the state terms (for ro_reward / rb_reward; n_state of them) and the joint state-action terms (for the *_joint
// kernels), each in term order and padded with empty terms to 8; returns the number of joint terms
static inline int ro_split_rewards(const pilco_rollout* ro, int* n_state, pilco_reward_term state[8],
                                   pilco_reward_term joint[8]) {
    int n_joint = 0;
    *n_state = 0;
    for (int k = 0; k < 8; ++k) state[k] = joint[k] = pilco_reward_term();
    for (int k = 0; k < ro->n_rewards; ++k) {
        if (reward_on_joint(ro->rewards[k].kind)) joint[n_joint++] = ro->rewards[k];
        else state[(*n_state)++] = ro->rewards[k];
    }
    return n_joint;
}

// parameters of the forward cascade's per-step and reward kernels (rollout.cu)
struct RoDev {
    int R, H, Ds, U, t;
    int pol_kind, squash;
    const double* maxa;
    const double* W; long long W_bs; const double* b; long long b_bs;
    int n_rewards; pilco_reward_term rewards[8];
    const double* m0; long long m0_bs; const double* S0; long long S0_bs;
    double* traj_m; double* traj_S; double* reward; double* step_reward;
    double* risk; double* step_risk; double mult_mu; int n_mult;     // MULT channel (SafePILCO): risk[t*R + r]
    double* rew;                                                      // additive channel per step: rew[t*R + r]
    // per-step slots [R, len] for step t (cur) and t-1 (prev)
    double *mj, *sj, *Mp, *Sp, *Vp, *Mu, *Su, *Cq, *Vu;
    double *mj_prev, *sj_prev, *Md_prev, *Sd_prev, *Vd_prev;
    MMParams dyn_prev;        // finish of the dynamics MM launched at step t-1
    MMParams pol;             // finish of the policy MM launched at step t (RBF)
};

// parameters of the cascade's per-step kernels on phi (rollout.cu): state Ds = dyn.E, policy input Dh = pol.Ds = Ds + A
struct TgDev {
    RoDev p;                  // p.Ds = Dh: the policy's input dimension; traj_m / traj_S / m0 / S0 in Ds
    TrigMap tm;
    double *mh, *Sh, *Ch, *cx;        // slots of step t [R, len]
    const double* cx_prev;            // cx of step t-1
};

static inline int ro_count_mult(const pilco_rollout* ro) {
    int c = 0;
    for (int k = 0; k < ro->n_rewards; ++k) c += ro->rewards[k].channel == PILCO_CHANNEL_MULT;
    return c;
}

// the per-step state kernel of the noisy cascade (rollout_noise.cu; in place of tg_state): glue as tg_state, then both
// feature-moment sets, the linear policy at the noisy one, squash, the joint and cx at the true one; var the noise
// variances [MAXD], mz / Sz the slots of step t
int nz_state_launch(const TgDev& g, const double* var, double* mz, double* Sz, cudaStream_t st);
// the exploration objective's forward launches (rollout_explore.cu), after the reward launches in place of
// ro_reward_sum: ro_reward_var with the state terms' ds (state dimension ds.Ds) and, when dj is non-NULL,
// ro_reward_joint_var with the joint terms' dj (dimension dj->Ds + dj->U; dj->mj, dj->sj the joint Gaussians of step
// 0), into sigma_t^2 var [H][R]; then ro_reward_explore_sum with step_var [R][H] if set
int ex_reward_var_launch(const RoDev& ds, const RoDev* dj, double b, double* var, double* step_var, cudaStream_t st);
