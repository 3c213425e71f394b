// rollout.cuh -- workspace layout of the H-step cascade shared by rollout.cu and rollout_bwd.cu.
#pragma once
#include "mm_kernels.cuh"

struct RoWs {                 // offsets in doubles
    size_t mj, sj, Md, Sd, Vd, Mp, Sp, Vp, Mu, Su, Cq, Vu, risk, rew, dynws, polws, total;
};

static inline RoWs ro_ws_layout(const pilco_rollout* ro) {
    const size_t R = ro->R, H = ro->H;
    const size_t Ds = ro->pol.Ds, U = ro->pol.U, D = Ds + U, E = Ds;
    RoWs L; size_t o = 0;
    auto take = [&](size_t len) { size_t at = o; o += (H * R * len + 1) & ~(size_t)1; return at; };
    L.mj = take(D); L.sj = take(D * D);
    L.Md = take(E); L.Sd = take(E * E); L.Vd = take(D * E);
    L.Mp = take(U); L.Sp = take(U * U); L.Vp = take(Ds * U);
    L.Mu = take(U); L.Su = take(U * U); L.Cq = take(U * U); L.Vu = take(Ds * U);
    L.risk = take(1);                       // per-step risk of the MULT reward channel, [H][R]
    L.rew = take(1);                        // per-step additive reward, [H][R] (summed in step order by ro_reward_sum_kernel)
    L.dynws = o; o += pilco_mm_workspace_bytes(ro->dyn.n, ro->dyn.D, ro->dyn.E, ro->R) / 8;
    L.polws = o;
    if (ro->pol.kind == PILCO_POLICY_RBF)
        o += pilco_mm_workspace_bytes(ro->pol.rbf.n, ro->pol.rbf.D, ro->pol.rbf.E, ro->R) / 8;
    L.total = o;
    return L;
}

int ro_check(const pilco_rollout* ro);

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

// Optional hook of the forward (pilco_rollout_explore_forward): run after the reward launches in place of ro_reward_sum,
// with the state terms' parameters ds (state dimension ds.Ds) and, when a joint state-action term is present, the joint
// terms' dj (dimension dj->Ds + dj->U; dj->mj, dj->sj the joint Gaussians of step 0), else NULL.
typedef int (*RoRewardHook)(const RoDev& ds, const RoDev* dj, cudaStream_t st, const void* ctx);
struct NzFwd;
// pilco_rollout_angles_forward (ang may be NULL) with the hook above; hook == NULL is that call.  nz: measurement noise at
// the policy's input (pilco_rollout_noisy_forward, validated by the caller), NULL without.
int ro_forward_run(const pilco_rollout* ro, const pilco_angles* ang, RoRewardHook hook, const void* ctx, cudaStream_t st,
                   const NzFwd* nz = nullptr);

// ---- angular state dimensions (pilco_rollout_angles_*): state Ds = dyn.E, policy input Dh = pol.Ds = Ds + A ----
#include "trig_math.cuh"
// validation of a rollout with angles; fills tm.  PILCO_OK with tm.A == 0 when there are none.
int tg_check(const pilco_rollout* ro, const pilco_angles* ang, TrigMap* tm);

// parameters of the angle cascade's per-step kernels (rollout.cu)
struct TgDev {
    RoDev p;                  // p.Ds = Dh: the policy's input dimension; traj_m / traj_S / m0 / S0 in Ds
    TrigMap tm;
    double *mh, *Sh, *Ch, *cx;        // slots of step t [R, len]
    const double* cx_prev;            // cx of step t-1
};

struct TgWs {                 // offsets in doubles: ro_ws_layout's slots at the policy dimension Dh, plus per step
    RoWs b;                   // (m^, S^, C^) of the feature map and cx = cov(x, [phi, u]) [Ds, Dh + U]
    size_t mh, Sh, Ch, cx, total;
};

static inline TgWs tg_ws_layout(const pilco_rollout* ro) {
    const size_t R = ro->R, H = ro->H;
    const size_t Dh = ro->pol.Ds, U = ro->pol.U, D = Dh + U, E = ro->dyn.E;
    TgWs T; RoWs& L = T.b; size_t o = 0;
    auto take = [&](size_t len) { size_t at = o; o += (H * R * len + 1) & ~(size_t)1; return at; };
    L.mj = take(D); L.sj = take(D * D);
    L.Md = take(E); L.Sd = take(E * E); L.Vd = take(D * E);
    L.Mp = take(U); L.Sp = take(U * U); L.Vp = take(Dh * U);
    L.Mu = take(U); L.Su = take(U * U); L.Cq = take(U * U); L.Vu = take(Dh * U);
    L.risk = take(1); L.rew = take(1);
    T.mh = take(Dh); T.Sh = take(Dh * Dh); T.Ch = take(E * Dh); T.cx = take(E * D);
    L.dynws = o; o += pilco_mm_workspace_bytes(ro->dyn.n, ro->dyn.D, ro->dyn.E, ro->R) / 8;
    L.polws = o;
    if (ro->pol.kind == PILCO_POLICY_RBF)
        o += pilco_mm_workspace_bytes(ro->pol.rbf.n, ro->pol.rbf.D, ro->pol.rbf.E, ro->R) / 8;
    L.total = T.total = o;
    return T;
}
static inline int ro_count_mult(const pilco_rollout* ro) {
    int c = 0;
    for (int k = 0; k < ro->n_rewards; ++k) c += ro->rewards[k].channel == PILCO_CHANNEL_MULT;
    return c;
}

// ---- measurement noise at the policy's input (pilco_rollout_noisy_*, rollout_noise.cu) ----
// The angle cascade (A >= 0; with A = 0 phi is the identity) whose policy reads the moments (m^_z, S^_z) of phi under
// N(m, S + diag(var)), kept per step after the angle layout (and before the exploration slot, when there is one).
struct NzFwd {
    double var[MAXD];         // noise variance of each raw state dimension
    size_t mz, Sz;            // offsets in doubles in ro->ws: [H][R][Dh], [H][R][Dh][Dh]
};

// the angle layout, then the noisy moments; `total` is where an exploration slot would go
static inline NzFwd nz_ws_layout(const pilco_rollout* ro, size_t* total) {
    const size_t R = ro->R, H = ro->H, Dh = ro->pol.Ds;
    NzFwd L;
    size_t o = tg_ws_layout(ro).total;
    auto take = [&](size_t len) { size_t at = o; o += (H * R * len + 1) & ~(size_t)1; return at; };
    L.mz = take(Dh); L.Sz = take(Dh * Dh);
    *total = o;
    return L;
}

// the per-step state kernel of the noisy cascade (in place of tg_state): glue as tg_state, then both feature-moment
// sets, the linear policy at the noisy one, squash, the joint and cx at the true one; mz / Sz the slots of step t
int nz_state_launch(const TgDev& g, const NzFwd& nz, double* mz, double* Sz, cudaStream_t st);
