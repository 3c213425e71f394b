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

// ---- angular state dimensions (pilco_rollout_angles_*): state Ds = dyn.E, policy input Dh = pol.Ds = Ds + A ----
#include "trig_math.cuh"
// validation of a rollout with angles; fills tm.  PILCO_OK with tm.A == 0 when there are none.
int tg_check(const pilco_rollout* ro, const pilco_angles* ang, TrigMap* tm);

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
