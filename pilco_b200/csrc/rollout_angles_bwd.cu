// rollout_angles_bwd.cu -- reverse sweep of the H-step cascade with angular state dimensions
// (pilco_rollout_angles_backward).  A translation unit of its own, so that the kernels of rollout_bwd.cu compile
// exactly as they do without it.
#include "mm_backward.cuh"
#include "mm_tape.cuh"
#include "rollout_bwd.cuh"
#include "small_kernels.cuh"

extern "C" size_t pilco_mm_bwd_workspace_bytes(int n, int D, int E, int R, int need_param);
void chol_solve_vec_launch(cudaStream_t st, int batch, int n, const double* L, int ld, long long ms, int E,
                           const double* Y, long long Y_bs, long long y_es, int yinc, double* x, long long xs);

// ---------------------------------------------------------------------------------------------
// Reverse sweep with angular state dimensions (pilco_rollout_angles_backward).  (gm, gS) is the cotangent of the raw
// state; the glue S' = S_x + S_d + cx V_d + (cx V_d)^T, cx = S_x C^ [I, V_u], seeds the dynamics VJP with
// gM = gm, gS = gS, gV = cx^T (gS + gS^T) and hands gcx = (gS + gS^T) V_d^T to the post stage.  Per step t:
//   taped:      tg_dyn_finish<DP> (mm_tape_bfinish_task with the explicit gV; last CTA of a restart: tg_post)
//   recomputing: mm_backward (dynamics) -> tg_post
//   tg_post: joint VJP on (m^, S^, V_u) + the cx cotangent (split over S_x, C^ and V_u), squash and linear-policy VJPs
//            at dimension Dh, into the feature cotangent (gm^, gS^, gC^)
//   RBF policy: mm_backward (policy, accumulating into (gm^, gS^))
//   tg_trig: dev_trig_bwd into (gm, gS), the state reward gradients, and the seeds gV, gcx of step t-1 (a kernel of
//            its own: folded into tg_post it made that kernel spill)
// ---------------------------------------------------------------------------------------------
struct TbWs {            // offsets in doubles
    size_t gm, gS, gVd, gcx, gmj, gsj, gMp, gSp, gVp, gmh, gSh, gCh, gbeta, gy, rgm, rgS, jgm, jgS, cnt, dynb, polb, total;
};

static TbWs tb_ws_layout(const pilco_rollout* ro) {
    const size_t R = ro->R, H = ro->H, Dh = ro->pol.Ds, U = ro->pol.U, D = Dh + U, Ds = ro->dyn.E;
    TbWs L; size_t o = 0;
    auto take = [&](size_t len) { size_t at = o; o += (R * len + 1) & ~(size_t)1; return at; };
    L.gm = take(Ds); L.gS = take(Ds * Ds); L.gVd = take(D * Ds); L.gcx = take(Ds * D);
    L.gmj = take(D); L.gsj = take(D * D);
    L.gMp = take(U); L.gSp = take(U * U); L.gVp = take(Dh * U);
    L.gmh = take(Dh); L.gSh = take(Dh * Dh); L.gCh = take(Ds * Dh);
    const size_t bf = ro->pol.kind == PILCO_POLICY_RBF ? ro->pol.rbf.n : 0;
    L.gbeta = take(U * bf); L.gy = take(U * bf);
    L.rgm = take(H * 2 * Ds); L.rgS = take(H * 2 * Ds * Ds);
    const size_t Hj = rb_has_joint(ro) ? H : 0;
    L.jgm = take(Hj * 2 * D); L.jgS = take(Hj * 2 * D * D);
    L.cnt = take(1);
    L.dynb = o;
    if (ro->tape) o += ((size_t)ro->R * mm_tape_bwd_part_doubles(ro->dyn.D, ro->dyn.E) + 1) & ~(size_t)1;
    else o += pilco_mm_bwd_workspace_bytes(ro->dyn.n, ro->dyn.D, ro->dyn.E, ro->R, 0) / 8;
    L.polb = o;
    if (ro->pol.kind == PILCO_POLICY_RBF)
        o += pilco_mm_bwd_workspace_bytes(ro->pol.rbf.n, ro->pol.rbf.D, ro->pol.rbf.E, ro->R, 1) / 8;
    L.total = o;
    return L;
}

struct TbPostSmem { SmallScratch sc; double gMu[MAXD], gSu[MAXD * MAXD], gVu[MAXD * MAXD], gB[MAXD * MAXD], gCd[MAXD],
                    gQ[MAXD * MAXD]; };

// trig VJP into the state cotangent, the state reward gradients of step t, then the seeds of step t-1
__global__ void __launch_bounds__(128) tg_trig_kernel(TbDev g) {
    PDL_ENTRY();
    const int r = blockIdx.x;
    const RbDev& p = g.p;
    const int Ds = g.tm.Ds, Dh = p.Ds, D = Dh + p.U, t = p.t;
    const int tid = threadIdx.x, nt = blockDim.x;
    double* gm = p.gm + (size_t)r * Ds;
    double* gS = p.gS + (size_t)r * Ds * Ds;
    const double* mx = p.traj_m + ((size_t)r * (p.H + 1) + t) * Ds;
    const double* sx = p.traj_S + ((size_t)r * (p.H + 1) + t) * Ds * Ds;
    dev_trig_bwd(g.tm, mx, sx, g.gmh + (size_t)r * Dh, g.gSh + (size_t)r * Dh * Dh, g.gCh + (size_t)r * Ds * Dh, gm, gS);
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

__device__ __forceinline__ void tg_post_body(const TbDev& g, int r, TbPostSmem& sm) {
    const RbDev& p = g.p;
    SmallScratch& sc = sm.sc;
    double* gMu = sm.gMu; double* gSu = sm.gSu; double* gVu = sm.gVu; double* gB = sm.gB; double* gCd = sm.gCd;
    double* gQ = sm.gQ;
    const int Ds = g.tm.Ds, Dh = p.Ds, U = p.U, D = Dh + U, t = p.t;
    const int tid = threadIdx.x, nt = blockDim.x;
    double* gS = p.gS + (size_t)r * Ds * Ds;
    if (p.tpart) {
        mm_tape_reduce_device(p.tpart + (size_t)r * p.tp_ntask * (MAXD + (size_t)D * D), p.tp_ntask, D,
                              p.gmj + (size_t)r * D, p.gsj + (size_t)r * D * D, 0);
        __syncthreads();
    }
    if (p.jgm) {
        double wmult = p.mult_mu;
        if (wmult != 0.0)
            for (int tt = 0; tt < p.H; ++tt) if (tt != t) wmult *= 1.0 - p.risk[(size_t)tt * p.R + r];
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
    const double* gcx = g.gcx + (size_t)r * Ds * D;
    const double* sx = p.traj_S + ((size_t)r * (p.H + 1) + t) * Ds * Ds;
    const double* mh = g.mh + (size_t)r * Dh;
    const double* Sh = g.Sh + (size_t)r * Dh * Dh;
    const double* Ch = g.Ch + (size_t)r * Ds * Dh;
    const double* cx = g.cx + (size_t)r * Ds * D;              // [Q, Q V_u]
    const double* Vu = p.Vu + (size_t)r * Dh * U;
    const double* Vp = p.Vp + (size_t)r * Dh * U;
    const double* Cq = p.Cq + (size_t)r * U * U;
    double* gmh = g.gmh + (size_t)r * Dh;
    double* gSh = g.gSh + (size_t)r * Dh * Dh;
    double* gCh = g.gCh + (size_t)r * Ds * Dh;
    // ---- joint VJP on (m^, S^, M_u, S_u, V_u) and the cross-covariance cotangent gcx = [gA, gB'] ----
    for (int e = tid; e < Dh * U; e += nt) {                 // gB = G12 + G21^T
        const int i = e / U, j = e % U;
        gB[e] = gsj[i * D + Dh + j] + gsj[(Dh + j) * D + i];
    }
    for (int i = tid; i < U; i += nt) gMu[i] = gmj[Dh + i];
    for (int e = tid; e < U * U; e += nt) gSu[e] = gsj[(Dh + e / U) * D + Dh + e % U];
    for (int e = tid; e < Ds * Dh; e += nt) {                // gQ = gA + gB' V_u^T
        const int i = e / Dh, k = e % Dh;
        double v = gcx[i * D + k];
        for (int j = 0; j < U; ++j) v = fma(gcx[i * D + Dh + j], Vu[k * U + j], v);
        gQ[e] = v;
    }
    __syncthreads();
    for (int i = tid; i < Dh; i += nt) gmh[i] = gmj[i];
    for (int e = tid; e < Dh * Dh; e += nt) {
        const int i = e / Dh, j = e % Dh;
        double v = gsj[i * D + j];
        for (int k = 0; k < U; ++k) v = fma(gB[i * U + k], Vu[j * U + k], v);       // gB V_u^T
        gSh[e] = v;
    }
    for (int e = tid; e < Dh * U; e += nt) {                 // gVu = S^^T gB + Q^T gB'
        const int i = e / U, j = e % U;
        double v = 0.0;
        for (int k = 0; k < Dh; ++k) v = fma(Sh[k * Dh + i], gB[k * U + j], v);
        for (int k = 0; k < Ds; ++k) v = fma(cx[k * D + i], gcx[k * D + Dh + j], v);
        gVu[e] = v;
    }
    for (int e = tid; e < Ds * Ds; e += nt) {                // gS_x += gQ C^^T   (cx = S_x C^ [I, V_u])
        const int i = e / Ds, j = e % Ds;
        double v = 0.0;
        for (int k = 0; k < Dh; ++k) v = fma(gQ[i * Dh + k], Ch[j * Dh + k], v);
        gS[e] += v;
    }
    for (int e = tid; e < Ds * Dh; e += nt) {                // gC^ = S_x^T gQ
        const int i = e / Dh, k = e % Dh;
        double v = 0.0;
        for (int l = 0; l < Ds; ++l) v = fma(sx[l * Ds + i], gQ[l * Dh + k], v);
        gCh[e] = v;
    }
    // the dynamics' direct cotangent of the state: gm_x += gm', gS_x += gS' (already in place: the glue's identity terms)
    __syncthreads();
    // ---- squash VJP:  V_u = V_p C ----
    double* gMp = p.gMp + (size_t)r * U;
    double* gSp = p.gSp + (size_t)r * U * U;
    double* gVp = p.gVp + (size_t)r * Dh * U;
    if (p.squash) {
        for (int k = tid; k < U; k += nt) {
            double v = 0.0;
            for (int i = 0; i < Dh; ++i) v = fma(Vp[i * U + k], gVu[i * U + k], v);
            gCd[k] = v;
        }
        for (int e = tid; e < Dh * U; e += nt) gVp[e] = gVu[e] * Cq[(e % U) * U + (e % U)];
        __syncthreads();
        dev_squash_bwd(U, p.Mp + (size_t)r * U, p.Sp + (size_t)r * U * U, p.maxa,
                       p.Mu + (size_t)r * U, p.Su + (size_t)r * U * U, gMu, gSu, gCd, gMp, gSp);
    } else {
        for (int i = tid; i < U; i += nt) gMp[i] = gMu[i];
        for (int e = tid; e < U * U; e += nt) gSp[e] = gSu[e];
        for (int e = tid; e < Dh * U; e += nt) gVp[e] = gVu[e];
        __syncthreads();
    }
    if (p.pol_kind == PILCO_POLICY_LINEAR) {
        dev_linear_bwd(Dh, U, p.W + (size_t)r * p.W_bs, mh, Sh, gMp, gSp, gVp,
                       p.gW + (size_t)r * U * Dh, p.gb + (size_t)r * U, gmh, gSh, sc);
    }
}

__global__ void __launch_bounds__(128) tg_post_kernel(TbDev g) {
    PDL_ENTRY();
    extern __shared__ __align__(16) unsigned char rb_dyn_smem[];
    tg_post_body(g, blockIdx.x, *reinterpret_cast<TbPostSmem*>(rb_dyn_smem));
}

template <int DP>
__global__ void __launch_bounds__(TB_THREADS, 3) tg_dyn_finish_kernel(MMTapeBwd bp, TbDev g) {
    PDL_ENTRY();
    extern __shared__ __align__(16) unsigned char rb_dyn_smem[];
    const int r = blockIdx.y;
    mm_tape_bfinish_task<DP>(bp, r, blockIdx.x, reinterpret_cast<double*>(rb_dyn_smem));
    if (last_cta_arrives(g.p.cnt + r, gridDim.x)) tg_post_body(g, r, *reinterpret_cast<TbPostSmem*>(rb_dyn_smem));
}

template <int DP>
static int launch_tg_dyn_finish(const MMTapeBwd& tb, const TbDev& g, cudaStream_t st) {
    size_t smem = mm_tape_bfinish_smem_bytes(tb.TL.np, tb.gp.D);
    if (smem < sizeof(TbPostSmem)) smem = sizeof(TbPostSmem);
    if (pilco_smem_optin<tg_dyn_finish_kernel<DP>>(196 * 1024)) return PILCO_ERR_LAUNCH;
    launch_hi(tg_dyn_finish_kernel<DP>, dim3(tb.gp.E + tb.TL.P, tb.R), dim3(TB_THREADS), smem, st, tb, g);
    return PILCO_OK;
}

extern "C" {

size_t pilco_rollout_angles_bwd_workspace_bytes(const pilco_rollout* ro, const pilco_angles* ang) {
    if (!ang || ang->A == 0) return pilco_rollout_bwd_workspace_bytes(ro);
    if (!ro || ro->R < 1 || ro->H < 0) return 0;
    return tb_ws_layout(ro).total * sizeof(double);
}

}  // extern "C"

// with measurement noise: the angle layout, then the cotangent of the noisy moments (gm^_z [R][Dh], gS^_z [R][Dh][Dh])
static size_t nz_bwd_layout(const pilco_rollout* ro, size_t* gmz, size_t* gSz) {
    const size_t R = ro->R, Dh = ro->pol.Ds;
    size_t o = tb_ws_layout(ro).total;
    *gmz = o; o += (R * Dh + 1) & ~(size_t)1;
    *gSz = o; o += (R * Dh * Dh + 1) & ~(size_t)1;
    return o;
}

size_t nz_bwd_ws_doubles(const pilco_rollout* ro) {
    size_t a, b;
    return nz_bwd_layout(ro, &a, &b);
}

int rb_backward_run(const pilco_rollout* ro, const pilco_angles* ang, const pilco_rollout_grad* g, RbRewardHook hook,
                    const void* ctx, cudaStream_t stream, const NzFwd* nz) {
    TrigMap tm;
    int rc = tg_check(ro, ang, &tm);
    if (rc) return rc;
    if (tm.A == 0 && !nz) return rb_backward_impl(ro, g, hook, ctx, stream);
    if (tm.A == 0) trig_map_make(ro->dyn.E, 0, nullptr, &tm);      // measurement noise without angles: phi = identity
    if (!g || !g->ws) return PILCO_ERR_NULL;
    const TgWs FT = tg_ws_layout(ro);
    const RoWs& FL = FT.b;
    const TbWs BL = tb_ws_layout(ro);
    size_t o_gmz = 0, o_gSz = 0;
    const size_t need = nz ? nz_bwd_layout(ro, &o_gmz, &o_gSz) : BL.total;
    if (g->ws_bytes < need * sizeof(double)) return PILCO_ERR_WORKSPACE;
    if (((uintptr_t)g->ws) & 15) return PILCO_ERR_ALIGN;
    const int R = ro->R, H = ro->H, Ds = tm.Ds, Dh = ro->pol.Ds, U = ro->pol.U, D = Dh + U;
    const bool rbf = ro->pol.kind == PILCO_POLICY_RBF;
    if (rbf) { if (!g->gXc || !g->gYc || !g->gell || !g->pol_L) return PILCO_ERR_NULL; }
    else { if (!g->gW || !g->gb) return PILCO_ERR_NULL; }
    cudaStream_t st = (cudaStream_t)stream;
    double* fws = (double*)ro->ws;
    double* bws = (double*)g->ws;
    const size_t RR = (size_t)R;
    auto slot = [&](size_t base, size_t len, int t) { return fws + base + (size_t)t * RR * len; };
    auto buf = [&](size_t base) { return bws + base; };

    // zero the state cotangent and the seeds of step H-1, the counters and the parameter-gradient accumulators
    cudaMemsetAsync(buf(BL.gm), 0, sizeof(double) * (BL.gmj - BL.gm), st);
    cudaMemsetAsync(buf(BL.cnt), 0, sizeof(double) * (BL.dynb - BL.cnt), st);
    const int bf = rbf ? ro->pol.rbf.n : 0;
    if (rbf) {
        cudaMemsetAsync(g->gXc, 0, sizeof(double) * RR * bf * Dh, st);
        cudaMemsetAsync(g->gell, 0, sizeof(double) * RR * U * Dh, st);
        cudaMemsetAsync(buf(BL.gbeta), 0, sizeof(double) * RR * U * bf, st);
    } else {
        cudaMemsetAsync(g->gW, 0, sizeof(double) * RR * U * Dh, st);
        cudaMemsetAsync(g->gb, 0, sizeof(double) * RR * U, st);
    }
    if (nz) cudaMemsetAsync(buf(o_gmz), 0, sizeof(double) * (need - o_gmz), st);     // nz_trig re-zeroes after each step
    if (!ro->tape) mm_bwd_zero_counters(mm_bws_layout(ro->dyn.n, ro->dyn.D, ro->dyn.E, 0), bws + BL.dynb, R, st);
    if (rbf) mm_bwd_zero_counters(mm_bws_layout(ro->pol.rbf.n, ro->pol.rbf.D, ro->pol.rbf.E, 1), bws + BL.polb, R, st);

    TbDev tg;
    tg.tm = tm;
    RbDev& d = tg.p;
    d.R = R; d.H = H; d.Ds = Dh; d.U = U;
    d.pol_kind = ro->pol.kind; d.squash = ro->pol.squash; d.maxa = ro->pol.max_action;
    d.W = ro->pol.W; d.W_bs = ro->pol.W_bs;
    int n_joint = 0;
    pilco_reward_term joint_terms[8];
    d.n_rewards = 0;
    for (int k = 0; k < 8; ++k) d.rewards[k] = joint_terms[k] = pilco_reward_term();
    for (int k = 0; k < ro->n_rewards; ++k) {
        if (reward_on_joint(ro->rewards[k].kind)) joint_terms[n_joint++] = ro->rewards[k];
        else d.rewards[d.n_rewards++] = ro->rewards[k];
    }
    d.traj_m = ro->traj_m; d.traj_S = ro->traj_S;
    d.risk = fws + FL.risk; d.mult_mu = ro_count_mult(ro) > 0 ? ro->mult_mu : 0.0;
    d.gm = buf(BL.gm); d.gS = buf(BL.gS); d.gMd = d.gSd = d.gVd = nullptr;
    d.gmj = buf(BL.gmj); d.gsj = buf(BL.gsj); d.gsjx = nullptr;
    d.gMp = buf(BL.gMp); d.gSp = buf(BL.gSp); d.gVp = buf(BL.gVp);
    d.gW = g->gW; d.gb = g->gb;
    d.rgm = buf(BL.rgm); d.rgS = buf(BL.rgS);
    const bool joint = rb_has_joint(ro);
    d.jgm = joint ? buf(BL.jgm) : nullptr; d.jgS = joint ? buf(BL.jgS) : nullptr;
    d.mj0 = fws + FL.mj; d.sj0 = fws + FL.sj;
    d.tpart = ro->tape ? bws + BL.dynb : nullptr;
    d.tp_ntask = ro->dyn.E + npairs_of(ro->dyn.E);
    d.cnt = reinterpret_cast<unsigned*>(buf(BL.cnt));
    d.t = 0;
    tg.gVd = buf(BL.gVd); tg.gcx = buf(BL.gcx); tg.gmh = buf(BL.gmh); tg.gSh = buf(BL.gSh); tg.gCh = buf(BL.gCh);
    double* gmz = nz ? buf(o_gmz) : nullptr;
    double* gSz = nz ? buf(o_gSz) : nullptr;
    if (H > 0) {
        d.sj = d.Vd = d.Mp = d.Sp = d.Vp = d.Mu = d.Su = d.Cq = d.Vu = nullptr;
        RbDev ds = d;                                 // the state terms at the raw trajectory
        ds.Ds = Ds;
        RbDev dj = d;                                 // the joint terms at [phi, u]: D = Dh + U
        dj.n_rewards = n_joint;
        for (int k = 0; k < 8; ++k) dj.rewards[k] = joint_terms[k];
        rc = rb_reward_launch(ds, joint ? &dj : nullptr, st);
        if (rc) return rc;
        if (hook) {
            rc = hook(ds, joint ? &dj : nullptr, st, ctx);
            if (rc) return rc;
        }
    }

    for (int t = H - 1; t >= 0; --t) {
        d.t = t;
        d.sj = slot(FL.sj, (size_t)D * D, t); d.Vd = slot(FL.Vd, (size_t)D * Ds, t);
        d.Mp = slot(FL.Mp, U, t); d.Sp = slot(FL.Sp, (size_t)U * U, t); d.Vp = slot(FL.Vp, (size_t)Dh * U, t);
        d.Mu = slot(FL.Mu, U, t); d.Su = slot(FL.Su, (size_t)U * U, t); d.Cq = slot(FL.Cq, (size_t)U * U, t);
        d.Vu = slot(FL.Vu, (size_t)Dh * U, t);
        tg.mh = slot(FT.mh, Dh, t); tg.Sh = slot(FT.Sh, (size_t)Dh * Dh, t); tg.Ch = slot(FT.Ch, (size_t)Ds * Dh, t);
        tg.cx = slot(FT.cx, (size_t)Ds * D, t);
        tg.cx_prev = t > 0 ? slot(FT.cx, (size_t)Ds * D, t - 1) : nullptr;
        tg.Vd_prev = t > 0 ? slot(FL.Vd, (size_t)D * Ds, t - 1) : nullptr;
        TbDev tp = tg;                                // with noise, the post stage stops before the linear-policy VJP,
        if (nz) tp.p.pol_kind = -1;                   // which nz_trig runs at the noisy moments
        if (ro->tape) {
            const MMTapeL TL = mm_tape_layout(ro->dyn.n, ro->dyn.D, ro->dyn.E, R);
            const MMTapeBwd tb = mm_tape_bwd_params(&ro->dyn, R, slot(FL.mj, D, t), D, slot(FL.sj, (size_t)D * D, t),
                                                    (long long)D * D, slot(FL.Md, Ds, t), d.gm, d.gS, tg.gVd,
                                                    (const double*)ro->tape + (size_t)t * RR * TL.per_r, TL,
                                                    bws + BL.dynb, d.gmj, D, d.gsj, (long long)D * D);
            rc = ks_dispatch(D, [&](auto ks) { return launch_tg_dyn_finish<4 * ks>(tb, tp, st); });
            if (rc) return rc;
            CUDA_LAUNCH_CHECK();
        } else {
            MMBwdParams bp = mm_bwd_params(&ro->dyn, R, slot(FL.mj, D, t), D, slot(FL.sj, (size_t)D * D, t), (long long)D * D,
                                           slot(FL.Md, Ds, t), d.gm, d.gS, tg.gVd,
                                           d.gmj, D, d.gsj, (long long)D * D, nullptr, nullptr, nullptr, 0, bws + BL.dynb);
            rc = mm_backward_launch(bp, st);
            if (rc) return rc;
            launch_hi(tg_post_kernel, dim3(R), dim3(128), sizeof(TbPostSmem), st, tp);
            CUDA_LAUNCH_CHECK();
        }
        const double* mz = nz ? slot(nz->mz, Dh, t) : nullptr;
        const double* Sz = nz ? slot(nz->Sz, (size_t)Dh * Dh, t) : nullptr;
        if (rbf) {                                    // the policy's input: the feature moments (the noisy ones with nz)
            MMBwdParams pp = mm_bwd_params(&ro->pol.rbf, R, nz ? mz : tg.mh, Dh, nz ? Sz : tg.Sh, (long long)Dh * Dh,
                                           slot(FL.Mp, U, t), d.gMp, d.gSp, d.gVp,
                                           nz ? gmz : tg.gmh, Dh, nz ? gSz : tg.gSh, (long long)Dh * Dh,
                                           g->gXc, buf(BL.gbeta), g->gell, 1, bws + BL.polb);
            rc = mm_backward_launch(pp, st);
            if (rc) return rc;
        }
        if (nz) {
            rc = nz_trig_launch(tg, *nz, mz, Sz, gmz, gSz, st);
            if (rc) return rc;
        } else {
            launch_hi(tg_trig_kernel, dim3(R), dim3(128), 0, st, tg);
            CUDA_LAUNCH_CHECK();
        }
    }
    if (rbf) {
        const int ldw = pad64(bf);
        chol_solve_vec_launch(st, R * U, bf, g->pol_L, ldw, (long long)ldw * ldw, U,
                              buf(BL.gbeta), (long long)U * bf, bf, 1, buf(BL.gy), bf);
        rc = rbf_factor_bwd_launch(st, R, bf, Dh, U, ro->pol.rbf.X, (long long)bf * Dh, ro->pol.rbf.ell, (long long)U * Dh,
                                   ro->pol.rbf.sf2, ro->pol.rbf.sf2_bs, ro->pol.rbf.beta, (long long)U * bf,
                                   buf(BL.gy), g->gXc, g->gYc, g->gell);
        if (rc) return rc;
    }
    if (g->gm0) cudaMemcpyAsync(g->gm0, d.gm, sizeof(double) * RR * Ds, cudaMemcpyDeviceToDevice, st);
    if (g->gS0) cudaMemcpyAsync(g->gS0, d.gS, sizeof(double) * RR * Ds * Ds, cudaMemcpyDeviceToDevice, st);
    return PILCO_OK;
}

extern "C" int pilco_rollout_angles_backward(const pilco_rollout* ro, const pilco_angles* ang, const pilco_rollout_grad* g,
                                             pilco_stream_t stream) {
    return rb_backward_run(ro, ang, g, nullptr, nullptr, (cudaStream_t)stream);
}
