// rollout_bwd.cu -- reverse sweep of the H-step cascade: d(sum_t E[r(x_t)]) / d(policy parameters).
// The reference obtains this gradient from TensorFlow autodiff through tf.while_loop
// (pilco/models/pilco.py:47-50, 84-90); here every stage has a hand-derived VJP (oracle/staged.py) and the
// forward's per-step joint Gaussians / policy moments saved by pilco_rollout_forward are re-used.
//
// The sweep is a strictly serial chain over the H steps, so its cost at small batches is (kernels per step) x
// (latency of each): the chain is kept short.
//   once      rb_reward  grid (R,H): d reward_t / d(m_t, S_t) of EVERY step -- it depends on the saved trajectory only;
//                        with joint state-action terms rb_reward_joint likewise: d reward_t / d(m~_t, s~_t) at the saved joint
//                        Gaussians, which rb_post adds to the joint's cotangent before the joint VJP hands it on
//   per step t = H-1 .. 0, with a tape (pilco_rollout.tape):
//     rb_dyn_finish  grid (E+P, R): tape-driven VJP of the dynamics moment match (mm_tape_bfinish_task; the glue seeds
//                    gM = gm, gS, gV = s1'(gS+gS') are formed inline); the LAST CTA of a restart to arrive then runs
//                    rb_post for it: sum of the task partials, joint / squash / linear-policy / reward VJPs ->
//                    state cotangent (gm_t, gS_t) and the seeds of the policy moment match
//     mm_backward (RBF policy, accumulating): fused setup -> btile -> bfinish(+reduce)        = 4 launches per step
//   without a tape (memory-lean): rb_pre -> mm_backward (dynamics, recomputing) -> rb_post -> mm_backward (policy)
// then, for the RBF policy, the VJP through beta = (K + sn2 I)^-1 Y.
#include "mm_backward.cuh"
#include "mm_tape.cuh"
#include "rollout.cuh"
#include "small_kernels.cuh"
#include "rollout_bwd.cuh"

extern "C" size_t pilco_mm_bwd_workspace_bytes(int n, int D, int E, int R, int need_param);
int chol_solve_vec_launch(cudaStream_t st, int batch, int n, const double* L, int ld, long long ms, int E,
                          const double* Y, long long Y_bs, long long y_es, int yinc, double* x, long long xs);

struct RbWs {            // backward workspace (offsets in doubles)
    size_t gm, gS, gMd, gSd, gVd, gcx, gmj, gsj, gsjx, gMp, gSp, gVp, gmh, gSh, gCh, gbeta, gy, rgm, rgS, jgm, jgS, cnt,
           dynb, polb, gmz, gSz, sgW, sgb, total;
};

// Dh = pol.Ds, Ds = dyn.E on phi (pol.Ds without).  Without phi the seeds of the dynamics VJP (gMd, gSd, gVd) and the
// glue's joint cotangent gsjx have slots of their own (rb_pre); on phi gVd and gcx are the seeds tg_trig leaves and
// (gmh, gSh, gCh) the feature cotangent; with noise (gmz, gSz) the cotangent of the noisy moments.  A slot whose
// feature is off has length 0.  An active policy schedule appends the per-step cotangents of W_t and b_t, step-major
// ([H][R][U*Dh], [H][R][U]: what rb_post / tg_post / nz_trig write at step t), after every other slot.
static RbWs rb_ws_layout(const pilco_rollout* ro, const pilco_angles* ang, const pilco_obs_noise* nz,
                         const pilco_policy_schedule* sch = nullptr) {
    const bool phi = ro_on_phi(ang, nz);
    const size_t R = ro->R, H = ro->H, Dh = ro->pol.Ds, U = ro->pol.U, D = Dh + U, Ds = phi ? (size_t)ro->dyn.E : Dh;
    const size_t F = phi ? 1 : 0, P = 1 - F, N = nz ? 1 : 0;
    RbWs L; size_t o = 0;
    auto take = [&](size_t len) { size_t at = o; o += (R * len + 1) & ~(size_t)1; return at; };
    L.gm = take(Ds); L.gS = take(Ds * Ds);
    L.gMd = take(P * Ds); L.gSd = take(P * Ds * Ds); L.gVd = take(D * Ds); L.gcx = take(F * Ds * D);
    L.gmj = take(D); L.gsj = take(D * D); L.gsjx = take(P * D * D);
    L.gMp = take(U); L.gSp = take(U * U); L.gVp = take(Dh * U);
    L.gmh = take(F * Dh); L.gSh = take(F * Dh * Dh); L.gCh = take(F * Ds * Dh);
    const size_t bf = ro->pol.kind == PILCO_POLICY_RBF ? ro->pol.rbf.n : 0;
    L.gbeta = take(U * bf); L.gy = take(U * bf);
    // reward gradients of every step, per channel (0: additive, 1: multiplicative): [H][2][R][Ds], [H][2][R][Ds*Ds]
    L.rgm = take(H * 2 * Ds); L.rgS = take(H * 2 * Ds * Ds);
    // likewise for the joint state-action terms, only when there is one: [H][2][R][D], [H][2][R][D*D]
    const size_t Hj = rb_has_joint(ro) ? H : 0;
    L.jgm = take(Hj * 2 * D); L.jgS = take(Hj * 2 * D * D);
    L.cnt = take(1);                                           // arrival counters of rb_dyn_finish (one per restart)
    // dynamics GP: task partials of the tape-driven reverse sweep, or the workspace of the recomputing one
    L.dynb = o;
    if (ro->tape) o += ((size_t)ro->R * mm_tape_bwd_part_doubles(ro->dyn.D, ro->dyn.E) + 1) & ~(size_t)1;
    else o += pilco_mm_bwd_workspace_bytes(ro->dyn.n, ro->dyn.D, ro->dyn.E, ro->R, 0) / 8;
    L.polb = o;
    if (ro->pol.kind == PILCO_POLICY_RBF)
        o += pilco_mm_bwd_workspace_bytes(ro->pol.rbf.n, ro->pol.rbf.D, ro->pol.rbf.E, ro->R, 1) / 8;
    L.gmz = take(N * Dh); L.gSz = take(N * Dh * Dh);
    const size_t HS = sch_active(sch) ? H : 0;
    L.sgW = take(HS * U * Dh); L.sgb = take(HS * U);
    L.total = o;
    return L;
}

// shared-memory scratch of rb_post_body (bytes), carved from a dynamic buffer
struct RbPostSmem { SmallScratch sc; double gMu[MAXD], gSu[MAXD * MAXD], gVu[MAXD * MAXD], gB[MAXD * MAXD], gCd[MAXD], gsjx[MAXD * MAXD]; };

// d (sum_k coef_k reward_k)(x_t) / d(m_t, S_t) for every step t and restart r, per accumulation channel
__global__ void __launch_bounds__(128) rb_reward_kernel(RbDev p) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    const int r = blockIdx.x, t = blockIdx.y, Ds = p.Ds;
    const int tid = threadIdx.x, nt = blockDim.x;
    const double* mx = p.traj_m + ((size_t)r * (p.H + 1) + t) * Ds;
    const double* sx = p.traj_S + ((size_t)r * (p.H + 1) + t) * Ds * Ds;
    double* gm0 = p.rgm + (((size_t)t * 2) * p.R + r) * Ds;
    double* gS0 = p.rgS + (((size_t)t * 2) * p.R + r) * Ds * Ds;
    double* gm1 = gm0 + (size_t)p.R * Ds;
    double* gS1 = gS0 + (size_t)p.R * Ds * Ds;
    for (int i = tid; i < Ds; i += nt) { gm0[i] = 0.0; gm1[i] = 0.0; }
    for (int e = tid; e < Ds * Ds; e += nt) { gS0[e] = 0.0; gS1[e] = 0.0; }
    __syncthreads();
    for (int k = 0; k < p.n_rewards; ++k) {
        const pilco_reward_term& rt = p.rewards[k];
        const bool mult = rt.channel == PILCO_CHANNEL_MULT;
        dev_reward_bwd(Ds, rt, mx, sx, rt.coef, mult ? gm1 : gm0, mult ? gS1 : gS0, sc);
    }
}

// the same for the joint state-action terms, at the forward's joint Gaussian (m~_t, s~_t) of every step: p.rewards holds
// those terms only, jgm / jgS their per-channel gradients [H][2][R][D], [H][2][R][D*D]
__global__ void __launch_bounds__(128) rb_reward_joint_kernel(RbDev p) {
    PDL_ENTRY();
    __shared__ SmallScratch sc;
    const int r = blockIdx.x, t = blockIdx.y, D = p.Ds + p.U;
    const int tid = threadIdx.x, nt = blockDim.x;
    const double* mj = p.mj0 + ((size_t)t * p.R + r) * D;
    const double* sj = p.sj0 + ((size_t)t * p.R + r) * D * D;
    double* gm0 = p.jgm + (((size_t)t * 2) * p.R + r) * D;
    double* gS0 = p.jgS + (((size_t)t * 2) * p.R + r) * D * D;
    double* gm1 = gm0 + (size_t)p.R * D;
    double* gS1 = gS0 + (size_t)p.R * D * D;
    for (int i = tid; i < D; i += nt) { gm0[i] = 0.0; gm1[i] = 0.0; }
    for (int e = tid; e < D * D; e += nt) { gS0[e] = 0.0; gS1[e] = 0.0; }
    __syncthreads();
    for (int k = 0; k < p.n_rewards; ++k) {
        const pilco_reward_term& rt = p.rewards[k];
        const bool mult = rt.channel == PILCO_CHANNEL_MULT;
        dev_joint_reward_bwd(D, rt, mj, sj, rt.coef, mult ? gm1 : gm0, mult ? gS1 : gS0, sc);
    }
}

__global__ void __launch_bounds__(128) rb_pre_kernel(RbDev p) {
    PDL_ENTRY();
    const int r = blockIdx.x, Ds = p.Ds, U = p.U, D = Ds + U;
    const int tid = threadIdx.x, nt = blockDim.x;
    const double* gm = p.gm + (size_t)r * Ds;
    const double* gS = p.gS + (size_t)r * Ds * Ds;
    const double* sj = p.sj + (size_t)r * D * D;
    const double* Vd = p.Vd + (size_t)r * D * Ds;
    for (int i = tid; i < Ds; i += nt) p.gMd[(size_t)r * Ds + i] = gm[i];
    for (int e = tid; e < Ds * Ds; e += nt) p.gSd[(size_t)r * Ds * Ds + e] = gS[e];
    // gVd = s1^T (gS + gS^T),   s1 = sj[:Ds, :]
    for (int e = tid; e < D * Ds; e += nt) {
        const int k = e / Ds, j = e % Ds;
        double v = 0.0;
        for (int i = 0; i < Ds; ++i) v = fma(sj[i * D + k], gS[i * Ds + j] + gS[j * Ds + i], v);
        p.gVd[(size_t)r * D * Ds + e] = v;
    }
    // extra cotangent of the joint covariance: rows < Ds get (gS + gS^T) Vd^T
    for (int e = tid; e < D * D; e += nt) {
        const int i = e / D, k = e % D;
        double v = 0.0;
        if (i < Ds) for (int j = 0; j < Ds; ++j) v = fma(gS[i * Ds + j] + gS[j * Ds + i], Vd[k * Ds + j], v);
        p.gsjx[(size_t)r * D * D + e] = v;
    }
}

// joint / squash / linear-policy / reward VJPs of step t for restart r (all 128 threads of one CTA)
__device__ __forceinline__ void rb_post_body(const RbDev& p, int r, RbPostSmem& sm) {
    SmallScratch& sc = sm.sc;
    double* gMu = sm.gMu; double* gSu = sm.gSu; double* gVu = sm.gVu; double* gB = sm.gB; double* gCd = sm.gCd;
    const int Ds = p.Ds, U = p.U, D = Ds + U, t = p.t;
    const int tid = threadIdx.x, nt = blockDim.x;
    double* gm = p.gm + (size_t)r * Ds;
    double* gS = p.gS + (size_t)r * Ds * Ds;
    const double* gsjx = p.gsjx + (size_t)r * D * D;
    if (p.tpart) {
        // taped dynamics VJP: sum its task partials (mm_tape_breduce folded in) and form the glue cotangent
        // gsjx = [(gS + gS') Vd' ; 0] (rb_pre folded in) -- both read gS BEFORE this step's update below
        mm_tape_reduce_device(p.tpart + (size_t)r * p.tp_ntask * (MAXD + (size_t)D * D), p.tp_ntask, D,
                              p.gmj + (size_t)r * D, p.gsj + (size_t)r * D * D, 0);
        const double* Vd = p.Vd + (size_t)r * D * Ds;
        for (int e = tid; e < D * D; e += nt) {
            const int i = e / D, k = e % D;
            double v = 0.0;
            if (i < Ds) for (int j = 0; j < Ds; ++j) v = fma(gS[i * Ds + j] + gS[j * Ds + i], Vd[k * Ds + j], v);
            sm.gsjx[e] = v;
        }
        gsjx = sm.gsjx;
        __syncthreads();
    }
    // MULT channel (safe_pilco.py:44-49): d[mu (1 - prod_t' (1 - risk_t'))] / d risk_t = mu prod_{t' != t} (1 - risk_t')
    double wmult = p.mult_mu;
    if (wmult != 0.0)
        for (int tt = 0; tt < p.H; ++tt) if (tt != t) wmult *= 1.0 - p.risk[(size_t)tt * p.R + r];
    if (p.jgm) {
        // joint state-action terms: their gradients at (m~_t, s~_t) join the cotangent the dynamics VJP left, with the
        // state terms' per-channel weights, so the joint VJP below distributes them to (m_x, S_x) and the policy moments
        double* gmj_w = p.gmj + (size_t)r * D;
        double* gsj_w = p.gsj + (size_t)r * D * D;
        const double* ja_m = p.jgm + (((size_t)t * 2) * p.R + r) * D;
        const double* ja_S = p.jgS + (((size_t)t * 2) * p.R + r) * D * D;
        const double* jm_m = ja_m + (size_t)p.R * D;
        const double* jm_S = ja_S + (size_t)p.R * D * D;
        for (int i = tid; i < D; i += nt) gmj_w[i] += ja_m[i] + wmult * jm_m[i];
        for (int e = tid; e < D * D; e += nt) gsj_w[e] += ja_S[e] + wmult * jm_S[e];
        __syncthreads();
    }
    const double* gmj = p.gmj + (size_t)r * D;
    const double* gsj = p.gsj + (size_t)r * D * D;
    const double* mx = p.traj_m + ((size_t)r * (p.H + 1) + t) * Ds;
    const double* sx = p.traj_S + ((size_t)r * (p.H + 1) + t) * Ds * Ds;
    const double* Vu = p.Vu + (size_t)r * Ds * U;
    const double* Vp = p.Vp + (size_t)r * Ds * U;
    const double* Cq = p.Cq + (size_t)r * U * U;
    // ---- joint VJP (pilco.py:141-144) ----
    for (int e = tid; e < Ds * U; e += nt) {                 // gB = G12 + G21^T
        const int i = e / U, j = e % U;
        gB[e] = gsj[i * D + Ds + j] + gsjx[i * D + Ds + j] + gsj[(Ds + j) * D + i] + gsjx[(Ds + j) * D + i];
    }
    for (int i = tid; i < U; i += nt) gMu[i] = gmj[Ds + i];
    for (int e = tid; e < U * U; e += nt) {
        const int i = e / U, j = e % U;
        gSu[e] = gsj[(Ds + i) * D + Ds + j] + gsjx[(Ds + i) * D + Ds + j];
    }
    __syncthreads();
    for (int i = tid; i < Ds; i += nt) gm[i] += gmj[i];
    for (int e = tid; e < Ds * Ds; e += nt) {
        const int i = e / Ds, j = e % Ds;
        double v = gsj[i * D + j] + gsjx[i * D + j];
        for (int k = 0; k < U; ++k) v = fma(gB[i * U + k], Vu[j * U + k], v);       // gB Vu^T
        gS[e] += v;
    }
    for (int e = tid; e < Ds * U; e += nt) {                 // gVu = s_x^T gB
        const int i = e / U, j = e % U;
        double v = 0.0;
        for (int k = 0; k < Ds; ++k) v = fma(sx[k * Ds + i], gB[k * U + j], v);
        gVu[e] = v;
    }
    __syncthreads();
    // ---- squash VJP (controllers.py:13-36, 118-120):  Vu = Vp C ----
    double* gMp = p.gMp + (size_t)r * U;
    double* gSp = p.gSp + (size_t)r * U * U;
    double* gVp = p.gVp + (size_t)r * Ds * U;
    if (p.squash) {
        for (int k = tid; k < U; k += nt) {
            double v = 0.0;
            for (int i = 0; i < Ds; ++i) v = fma(Vp[i * U + k], gVu[i * U + k], v);
            gCd[k] = v;
        }
        for (int e = tid; e < Ds * U; e += nt) gVp[e] = gVu[e] * Cq[(e % U) * U + (e % U)];
        __syncthreads();
        dev_squash_bwd(U, p.Mp + (size_t)r * U, p.Sp + (size_t)r * U * U, p.maxa,
                       p.Mu + (size_t)r * U, p.Su + (size_t)r * U * U, gMu, gSu, gCd, gMp, gSp);
    } else {
        for (int i = tid; i < U; i += nt) gMp[i] = gMu[i];
        for (int e = tid; e < U * U; e += nt) gSp[e] = gSu[e];
        for (int e = tid; e < Ds * U; e += nt) gVp[e] = gVu[e];
        __syncthreads();
    }
    // ---- linear policy VJP (controllers.py:52-54) ----
    if (p.pol_kind == PILCO_POLICY_LINEAR) {
        dev_linear_bwd(Ds, U, p.W + (size_t)r * p.W_bs, mx, sx, gMp, gSp, gVp,
                       p.gW + (size_t)r * U * Ds, p.gb + (size_t)r * U, gm, gS, sc);
    }
    // ---- reward VJP at state t (pilco.py:133): precomputed per channel by rb_reward_kernel, weighted by wmult ----
    const double* ra_m = p.rgm + (((size_t)t * 2) * p.R + r) * Ds;
    const double* ra_S = p.rgS + (((size_t)t * 2) * p.R + r) * Ds * Ds;
    const double* rm_m = ra_m + (size_t)p.R * Ds;
    const double* rm_S = ra_S + (size_t)p.R * Ds * Ds;
    for (int i = tid; i < Ds; i += nt) gm[i] += ra_m[i] + wmult * rm_m[i];
    for (int e = tid; e < Ds * Ds; e += nt) gS[e] += ra_S[e] + wmult * rm_S[e];
}

__global__ void __launch_bounds__(128) rb_post_kernel(RbDev p) {
    PDL_ENTRY();
    extern __shared__ __align__(16) unsigned char rb_dyn_smem[];
    rb_post_body(p, blockIdx.x, *reinterpret_cast<RbPostSmem*>(rb_dyn_smem));
}

// taped path: dynamics VJP from the tape + (last CTA of the restart) rb_post, ONE launch per step
template <int DP>
__global__ void __launch_bounds__(TB_THREADS, 3) rb_dyn_finish_kernel(MMTapeBwd bp, RbDev d) {
    PDL_ENTRY();
    extern __shared__ __align__(16) unsigned char rb_dyn_smem[];
    const int r = blockIdx.y;
    mm_tape_bfinish_task<DP>(bp, r, blockIdx.x, reinterpret_cast<double*>(rb_dyn_smem));
    if (last_cta_arrives(d.cnt + r, gridDim.x)) rb_post_body(d, r, *reinterpret_cast<RbPostSmem*>(rb_dyn_smem));
}

template <int DP>
static int launch_dyn_finish(const MMTapeBwd& tb, const RbDev& d, cudaStream_t st) {
    size_t smem = mm_tape_bfinish_smem_bytes(tb.TL.np, tb.gp.D);
    if (smem < sizeof(RbPostSmem)) smem = sizeof(RbPostSmem);
    if (pilco_smem_optin<rb_dyn_finish_kernel<DP>>(196 * 1024)) return PILCO_ERR_LAUNCH;
    launch_hi(rb_dyn_finish_kernel<DP>, dim3(tb.gp.E + tb.TL.P, tb.R), dim3(TB_THREADS), smem, st, tb, d);
    return PILCO_OK;
}

// VJP through beta_a = (K_a + sn2 I)^-1 y_a for the RBF policy (sf2 frozen, controllers.py:91-93): given gy_a = (K_a+sn2 I)^-1 gbeta_a,
//   gY[:,a] = gy_a ;  gK = -gy beta^T ;  gX += ..., gell += ...   (oracle/staged.py: rbf_factor_backward)
// X, ell, sf2, beta: the policy's arrays with their per-restart strides; gy, gX, gY, gell: contiguous [R, ...]
__global__ void __launch_bounds__(128) rbf_factor_bwd_kernel(int bf, int Ds, int U, const double* X, long long X_bs,
                                                             const double* ell, long long ell_bs,
                                                             const double* sf2, long long sf2_bs,
                                                             const double* beta, long long beta_bs, const double* gy,
                                                             double* gX, double* gY, double* gell) {
    PDL_ENTRY();
    // one CTA per restart, thread n owns centre n: K[n][m] is evaluated once per (n, m, a)
    const int r = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const double* Xr = X + (size_t)r * X_bs;
    const double* lr = ell + (size_t)r * ell_bs;
    const double* br = beta + (size_t)r * beta_bs;
    const double* gr = gy + (size_t)r * U * bf;
    __shared__ double sgl[MAXD * 4], sglo[MAXD];
    for (int e = tid; e < bf * U; e += nt) { const int n = e / U, a = e % U; gY[(size_t)r * bf * U + e] = gr[a * bf + n]; }
    for (int a = 0; a < U; ++a) {
        double il2[MAXD], accl[MAXD];
        const double sfa = sf2[(size_t)r * sf2_bs + a];
#pragma unroll
        for (int d = 0; d < MAXD; ++d) { il2[d] = d < Ds ? 1.0 / (lr[a * Ds + d] * lr[a * Ds + d]) : 0.0; accl[d] = 0.0; }
        for (int n = tid; n < bf; n += nt) {
            double xn[MAXD], accx[MAXD];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) { xn[d] = d < Ds ? Xr[n * Ds + d] : 0.0; accx[d] = 0.0; }
            const double gyn = gr[a * bf + n], bn = br[a * bf + n];
            for (int m = 0; m < bf; ++m) {
                double diff[MAXD], d2 = 0.0;
#pragma unroll
                for (int d = 0; d < MAXD; ++d) {
                    diff[d] = d < Ds ? xn[d] - Xr[m * Ds + d] : 0.0;
                    d2 = fma(diff[d] * diff[d], il2[d], d2);
                }
                const double K = sfa * exp(-0.5 * d2);
                const double gK = -gyn * br[a * bf + m] * K;                // dL/dK[n][m] * K
                const double Psym = gK - gr[a * bf + m] * bn * K;          // (gK + gK^T)[n][m] * K
#pragma unroll
                for (int d = 0; d < MAXD; ++d) {
                    accx[d] = fma(-Psym * il2[d], diff[d], accx[d]);
                    accl[d] = fma(gK, diff[d] * diff[d], accl[d]);
                }
            }
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < Ds) gX[(size_t)r * bf * Ds + n * Ds + d] += accx[d];
        }
        block_sum<MAXD>(accl, MAXD, sgl, sglo);
        if (tid < Ds) { const double l = lr[a * Ds + tid]; gell[(size_t)r * U * Ds + a * Ds + tid] += sglo[tid] / (l * l * l); }
        __syncthreads();
    }
}

// rbf_factor_bwd_kernel for callers in other translation units (the particle gradient, particles.cu)
int rbf_factor_bwd_launch(cudaStream_t st, int R, int bf, int Ds, int U, const double* X, long long X_bs,
                          const double* ell, long long ell_bs, const double* sf2, long long sf2_bs,
                          const double* beta, long long beta_bs, const double* gy,
                          double* gX, double* gY, double* gell) {
    launch_hi(rbf_factor_bwd_kernel, dim3(R), dim3(128), 0, st, bf, Ds, U, X, X_bs, ell, ell_bs, sf2, sf2_bs, beta, beta_bs,
              gy, gX, gY, gell);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int rb_reward_launch(const RbDev& ds, const RbDev* dj, cudaStream_t st) {
    launch_hi(rb_reward_kernel, dim3(ds.R, ds.H), dim3(128), 0, st, ds);
    CUDA_LAUNCH_CHECK();
    if (dj) {
        launch_hi(rb_reward_joint_kernel, dim3(dj->R, dj->H), dim3(128), 0, st, *dj);
        CUDA_LAUNCH_CHECK();
    }
    return PILCO_OK;
}

// the per-step policy cotangents, step-major in the workspace ([H][R][n]), to the caller's restart-major [R][H][n]
__global__ void __launch_bounds__(128) rb_sched_grad_kernel(int R, int H, int n, const double* __restrict__ src,
                                                             double* __restrict__ dst) {
    PDL_ENTRY();
    const size_t total = (size_t)R * H * n;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const size_t i = e % n, rt = e / n, t = rt % H, r = rt / H;
        dst[e] = src[(t * R + r) * n + i];
    }
}

static int rb_sched_grad_launch(int R, int H, int n, const double* src, double* dst, cudaStream_t st) {
    const size_t total = (size_t)R * H * n;
    if (total == 0) return PILCO_OK;
    const unsigned blocks = (unsigned)((total + 127) / 128 < 1024 ? (total + 127) / 128 : 1024);
    launch_hi(rb_sched_grad_kernel, dim3(blocks), dim3(128), 0, st, R, H, n, src, dst);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

// rb_post for step d.t: with a tape (tb) fused into rb_dyn_finish, the tape-driven dynamics VJP, else a launch of its own
static int rb_post_launch(const RbDev& d, const MMTapeBwd* tb, cudaStream_t st) {
    if (tb) {
        const int rc = ks_dispatch(d.Ds + d.U, [&](auto ks) { return launch_dyn_finish<4 * ks>(*tb, d, st); });
        if (rc) return rc;
    } else {
        launch_hi(rb_post_kernel, dim3(d.R), dim3(128), sizeof(RbPostSmem), st, d);
    }
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

// The reverse sweep of every call (ang, ex, nz, sch may be NULL).  Per step the post stage is rb_post (rb_pre before the
// recomputing dynamics VJP) or tg_post on phi, which with noise stops before the linear-policy VJP; the policy GP's
// VJP reads x_t, phi's moments or the noisy ones; the trig stage (on phi) is tg_trig or, with noise, nz_trig.
// With an active schedule the linear-policy VJP of step t reads W_t and accumulates into step t's own gradient slots
// (rb_ws_layout's sgW, sgb), which rb_sched_grad reorders into g->gW, g->gb after the sweep.
static int rb_backward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                       const pilco_obs_noise* nz, const pilco_policy_schedule* sch, const pilco_rollout_grad* g,
                       cudaStream_t st) {
    RoOpt o;
    int rc = ro_validate(ro, ang, ex, nz, true, &o, sch);
    if (rc) return rc;
    if (!g || !g->ws) return PILCO_ERR_NULL;
    const RbWs BL = rb_ws_layout(ro, ang, nz, sch);
    if (g->ws_bytes < BL.total * sizeof(double)) return PILCO_ERR_WORKSPACE;
    if (((uintptr_t)g->ws) & 15) return PILCO_ERR_ALIGN;
    const int R = ro->R, H = ro->H, Ds = ro->dyn.E, Dh = ro->pol.Ds, U = ro->pol.U, D = Dh + U;
    const bool rbf = ro->pol.kind == PILCO_POLICY_RBF;
    if (rbf) { if (!g->gXc || !g->gYc || !g->gell || !g->pol_L) return PILCO_ERR_NULL; }
    else { if (!g->gW || !g->gb) return PILCO_ERR_NULL; }
    const RoWs FL = ro_ws_layout(ro, ang, ex, nz);
    double* fws = (double*)ro->ws;
    double* bws = (double*)g->ws;
    const size_t RR = (size_t)R;
    auto slot = [&](size_t base, size_t len, int t) { return fws + base + (size_t)t * RR * len; };
    auto buf = [&](size_t base) { return bws + base; };

    // zero the state cotangent (on phi with the seeds of step H-1), the parameter-gradient accumulators and the arrival
    // counters
    cudaMemsetAsync(buf(BL.gm), 0, sizeof(double) * ((o.phi ? BL.gmj : BL.gMd) - BL.gm), st);
    cudaMemsetAsync(buf(BL.cnt), 0, sizeof(double) * (BL.dynb - BL.cnt), st);
    const int bf = rbf ? ro->pol.rbf.n : 0;
    if (rbf) {
        cudaMemsetAsync(g->gXc, 0, sizeof(double) * RR * bf * Dh, st);
        cudaMemsetAsync(g->gell, 0, sizeof(double) * RR * U * Dh, st);
        cudaMemsetAsync(buf(BL.gbeta), 0, sizeof(double) * RR * U * bf, st);
    } else if (sch_active(sch)) {
        cudaMemsetAsync(buf(BL.sgW), 0, sizeof(double) * (BL.total - BL.sgW), st);
    } else {
        cudaMemsetAsync(g->gW, 0, sizeof(double) * RR * U * Dh, st);
        cudaMemsetAsync(g->gb, 0, sizeof(double) * RR * U, st);
    }
    if (o.noise) cudaMemsetAsync(buf(BL.gmz), 0, sizeof(double) * (BL.total - BL.gmz), st);   // nz_trig re-zeroes
    // arrival counters of the finish kernels (self-cleaning afterwards): zero once per reverse sweep
    if (!ro->tape) mm_bwd_zero_counters(mm_bws_layout(ro->dyn.n, ro->dyn.D, ro->dyn.E, 0), bws + BL.dynb, R, st);
    if (rbf) mm_bwd_zero_counters(mm_bws_layout(ro->pol.rbf.n, ro->pol.rbf.D, ro->pol.rbf.E, 1), bws + BL.polb, R, st);

    TbDev tg;
    tg.tm = o.tm;
    RbDev& d = tg.p;
    d.R = R; d.H = H; d.Ds = Dh; d.U = U;
    d.pol_kind = ro->pol.kind; d.squash = ro->pol.squash; d.maxa = ro->pol.max_action;
    d.W = ro->pol.W; d.W_bs = ro->pol.W_bs;
    pilco_reward_term joint_terms[8];
    const int n_joint = ro_split_rewards(ro, &d.n_rewards, d.rewards, joint_terms);
    d.traj_m = ro->traj_m; d.traj_S = ro->traj_S;
    d.risk = fws + FL.risk; d.mult_mu = ro_count_mult(ro) > 0 ? ro->mult_mu : 0.0;
    d.gm = buf(BL.gm); d.gS = buf(BL.gS); d.gMd = buf(BL.gMd); d.gSd = buf(BL.gSd); d.gVd = buf(BL.gVd);
    d.gmj = buf(BL.gmj); d.gsj = buf(BL.gsj); d.gsjx = buf(BL.gsjx);
    d.gMp = buf(BL.gMp); d.gSp = buf(BL.gSp); d.gVp = buf(BL.gVp);
    d.gW = g->gW; d.gb = g->gb;
    d.rgm = buf(BL.rgm); d.rgS = buf(BL.rgS);
    const bool joint = n_joint > 0;
    d.jgm = joint ? buf(BL.jgm) : nullptr; d.jgS = joint ? buf(BL.jgS) : nullptr;
    d.mj0 = fws + FL.mj; d.sj0 = fws + FL.sj;
    d.tpart = ro->tape ? bws + BL.dynb : nullptr;
    d.tp_ntask = ro->dyn.E + npairs_of(ro->dyn.E);
    d.cnt = reinterpret_cast<unsigned*>(buf(BL.cnt));
    d.t = 0;
    tg.gVd = d.gVd; tg.gcx = buf(BL.gcx); tg.gmh = buf(BL.gmh); tg.gSh = buf(BL.gSh); tg.gCh = buf(BL.gCh);
    double* gmz = buf(BL.gmz);
    double* gSz = buf(BL.gSz);
    if (H > 0) {                                      // reward gradients of every step at once
        d.sj = d.Vd = d.Mp = d.Sp = d.Vp = d.Mu = d.Su = d.Cq = d.Vu = nullptr;
        RbDev ds = d;                                 // the state terms at the raw trajectory
        ds.Ds = Ds;
        RbDev dj = d;                                 // the joint terms at [phi, u]: D = Dh + U
        dj.n_rewards = n_joint;
        for (int k = 0; k < 8; ++k) dj.rewards[k] = joint_terms[k];
        rc = rb_reward_launch(ds, joint ? &dj : nullptr, st);
        if (rc) return rc;
        if (o.explore && o.b != 0.0) {
            rc = rb_reward_var_launch(ds, joint ? &dj : nullptr, o.b, fws + FL.var, st);
            if (rc) return rc;
        }
    }

    const long long W_ts = sch_active(sch) ? sch->W_ts : 0, b_ts = sch_active(sch) ? sch->b_ts : 0;
    for (int t = H - 1; t >= 0; --t) {
        d.t = t;
        if (W_ts || b_ts) {
            d.W = ro->pol.W + t * W_ts;
            d.gW = buf(BL.sgW) + (size_t)t * RR * U * Dh; d.gb = buf(BL.sgb) + (size_t)t * RR * U;
        }
        d.sj = slot(FL.sj, (size_t)D * D, t); d.Vd = slot(FL.Vd, (size_t)D * Ds, t);
        d.Mp = slot(FL.Mp, U, t); d.Sp = slot(FL.Sp, (size_t)U * U, t); d.Vp = slot(FL.Vp, (size_t)Dh * U, t);
        d.Mu = slot(FL.Mu, U, t); d.Su = slot(FL.Su, (size_t)U * U, t); d.Cq = slot(FL.Cq, (size_t)U * U, t);
        d.Vu = slot(FL.Vu, (size_t)Dh * U, t);
        tg.mh = slot(FL.mh, Dh, t); tg.Sh = slot(FL.Sh, (size_t)Dh * Dh, t); tg.Ch = slot(FL.Ch, (size_t)Ds * Dh, t);
        tg.cx = slot(FL.cx, (size_t)Ds * D, t);
        tg.cx_prev = t > 0 ? slot(FL.cx, (size_t)Ds * D, t - 1) : nullptr;
        tg.Vd_prev = t > 0 ? slot(FL.Vd, (size_t)D * Ds, t - 1) : nullptr;
        TbDev tp = tg;                                // with noise, the post stage stops before the linear-policy VJP,
        if (o.noise) tp.p.pol_kind = -1;              // which nz_trig runs at the noisy moments
        if (ro->tape) {                              // consume the tape of step t: no exponential is recomputed
            // seeds straight from the state cotangent (without phi gV = s1'(gS+gS') inline); tape slot (t, :)
            const MMTapeL TL = mm_tape_layout(ro->dyn.n, ro->dyn.D, ro->dyn.E, R);
            const MMTapeBwd tb = mm_tape_bwd_params(&ro->dyn, R, slot(FL.mj, D, t), D, slot(FL.sj, (size_t)D * D, t),
                                                    (long long)D * D, slot(FL.Md, Ds, t), d.gm, d.gS,
                                                    o.phi ? tg.gVd : nullptr,
                                                    (const double*)ro->tape + (size_t)t * RR * TL.per_r, TL,
                                                    bws + BL.dynb, d.gmj, D, d.gsj, (long long)D * D);
            rc = o.phi ? tg_post_launch(tp, &tb, st) : rb_post_launch(d, &tb, st);
            if (rc) return rc;
        } else {
            if (!o.phi) {
                launch_hi(rb_pre_kernel, dim3(R), dim3(128), 0, st, d);
                CUDA_LAUNCH_CHECK();
            }
            MMBwdParams bp = mm_bwd_params(&ro->dyn, R, slot(FL.mj, D, t), D, slot(FL.sj, (size_t)D * D, t), (long long)D * D,
                                           slot(FL.Md, Ds, t), o.phi ? d.gm : d.gMd, o.phi ? d.gS : d.gSd, d.gVd,
                                           d.gmj, D, d.gsj, (long long)D * D, nullptr, nullptr, nullptr, 0, bws + BL.dynb);
            rc = mm_backward_launch(bp, st);
            if (rc) return rc;
            rc = o.phi ? tg_post_launch(tp, nullptr, st) : rb_post_launch(d, nullptr, st);
            if (rc) return rc;
        }
        const double* mz = slot(FL.mz, Dh, t);
        const double* Sz = slot(FL.Sz, (size_t)Dh * Dh, t);
        if (rbf) {                                    // the policy's input: x_t, or phi's moments (the noisy ones)
            MMBwdParams pp = o.phi ? mm_bwd_params(&ro->pol.rbf, R, o.noise ? mz : tg.mh, Dh, o.noise ? Sz : tg.Sh,
                                                   (long long)Dh * Dh, slot(FL.Mp, U, t), d.gMp, d.gSp, d.gVp,
                                                   o.noise ? gmz : tg.gmh, Dh, o.noise ? gSz : tg.gSh, (long long)Dh * Dh,
                                                   g->gXc, buf(BL.gbeta), g->gell, 1, bws + BL.polb)
                                   : mm_bwd_params(&ro->pol.rbf, R, ro->traj_m + (size_t)t * Ds, (long long)(H + 1) * Ds,
                                                   ro->traj_S + (size_t)t * Ds * Ds, (long long)(H + 1) * Ds * Ds,
                                                   slot(FL.Mp, U, t), d.gMp, d.gSp, d.gVp,
                                                   d.gm, Dh, d.gS, (long long)Dh * Dh,
                                                   g->gXc, buf(BL.gbeta), g->gell, 1, bws + BL.polb);
            rc = mm_backward_launch(pp, st);
            if (rc) return rc;
        }
        if (o.noise) rc = nz_trig_launch(tg, o.nzvar, mz, Sz, gmz, gSz, st);
        else if (o.phi) rc = tg_trig_launch(tg, st);
        if (rc) return rc;
    }
    if (rbf) {
        // gy = (K + sn2 I)^-1 gbeta  with the Cholesky factors kept by pilco_gp_factorize
        const int ldw = pad64(bf);
        rc = chol_solve_vec_launch(st, R * U, bf, g->pol_L, ldw, (long long)ldw * ldw, U,
                                   buf(BL.gbeta), (long long)U * bf, bf, 1, buf(BL.gy), bf);
        if (rc) return rc;
        rc = rbf_factor_bwd_launch(st, R, bf, Dh, U, ro->pol.rbf.X, (long long)bf * Dh, ro->pol.rbf.ell, (long long)U * Dh,
                                   ro->pol.rbf.sf2, ro->pol.rbf.sf2_bs, ro->pol.rbf.beta, (long long)U * bf,
                                   buf(BL.gy), g->gXc, g->gYc, g->gell);
        if (rc) return rc;
    }
    if (W_ts || b_ts) {
        rc = rb_sched_grad_launch(R, H, U * Dh, buf(BL.sgW), g->gW, st);
        if (!rc) rc = rb_sched_grad_launch(R, H, U, buf(BL.sgb), g->gb, st);
        if (rc) return rc;
    }
    if (g->gm0) cudaMemcpyAsync(g->gm0, d.gm, sizeof(double) * RR * Ds, cudaMemcpyDeviceToDevice, st);
    if (g->gS0) cudaMemcpyAsync(g->gS0, d.gS, sizeof(double) * RR * Ds * Ds, cudaMemcpyDeviceToDevice, st);
    return PILCO_OK;
}

// the size of the reverse sweep's workspace (the exploration gradient adds none): 0 for a description without a batch
// or with H < 0
static size_t rb_ws_bytes(const pilco_rollout* ro, const pilco_angles* ang, const pilco_obs_noise* nz,
                          const pilco_policy_schedule* sch = nullptr) {
    if (!ro || ro->R < 1 || ro->H < 0 || (sch && (sch->W_ts < 0 || sch->b_ts < 0))) return 0;
    return rb_ws_layout(ro, ang, nz, sch).total * sizeof(double);
}

extern "C" {

size_t pilco_rollout_bwd_workspace_bytes(const pilco_rollout* ro) { return rb_ws_bytes(ro, nullptr, nullptr); }

size_t pilco_rollout_angles_bwd_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang) {
    return rb_ws_bytes(ro, ang, nullptr);
}

size_t pilco_rollout_explore_bwd_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang,
                                                 const pilco_exploration* ex) {
    (void)ex;
    return rb_ws_bytes(ro, ang, nullptr);
}

size_t pilco_rollout_noisy_bwd_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang,
                                               const pilco_exploration* ex, const pilco_obs_noise* nz) {
    (void)ex;
    return rb_ws_bytes(ro, ang, nz);
}

int pilco_rollout_backward(const pilco_rollout* ro, const pilco_rollout_grad* g, pilco_stream_t stream) {
    return rb_backward(ro, nullptr, nullptr, nullptr, nullptr, g, (cudaStream_t)stream);
}

int pilco_rollout_angles_backward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_rollout_grad* g,
                                  pilco_stream_t stream) {
    return rb_backward(ro, ang, nullptr, nullptr, nullptr, g, (cudaStream_t)stream);
}

int pilco_rollout_explore_backward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                   const pilco_rollout_grad* g, pilco_stream_t stream) {
    return rb_backward(ro, ang, ex, nullptr, nullptr, g, (cudaStream_t)stream);
}

int pilco_rollout_noisy_backward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                 const pilco_obs_noise* nz, const pilco_rollout_grad* g, pilco_stream_t stream) {
    return rb_backward(ro, ang, ex, nz, nullptr, g, (cudaStream_t)stream);
}

size_t pilco_rollout_scheduled_bwd_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang,
                                                   const pilco_exploration* ex, const pilco_obs_noise* nz,
                                                   const pilco_policy_schedule* sch) {
    (void)ex;
    return rb_ws_bytes(ro, ang, nz, sch);
}

int pilco_rollout_scheduled_backward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_exploration* ex,
                                     const pilco_obs_noise* nz, const pilco_policy_schedule* sch,
                                     const pilco_rollout_grad* g, pilco_stream_t stream) {
    return rb_backward(ro, ang, ex, nz, sch, g, (cudaStream_t)stream);
}

}  // extern "C"
