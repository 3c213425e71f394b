// rollout_angles_bwd.cu -- the per-step kernels of the reverse sweep on phi (angular state dimensions or measurement
// noise; the sweep itself is rollout_bwd.cu's).  A translation unit of its own, so that the kernels of rollout_bwd.cu
// compile exactly as they do without it.
#include "mm_backward.cuh"
#include "mm_tape.cuh"
#include "rollout_bwd.cuh"
#include "small_kernels.cuh"

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

int tg_post_launch(const TbDev& g, const MMTapeBwd* tb, cudaStream_t st) {
    if (tb) {
        const int rc = ks_dispatch(g.p.Ds + g.p.U, [&](auto ks) { return launch_tg_dyn_finish<4 * ks>(*tb, g, st); });
        if (rc) return rc;
    } else {
        launch_hi(tg_post_kernel, dim3(g.p.R), dim3(128), sizeof(TbPostSmem), st, g);
    }
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int tg_trig_launch(const TbDev& g, cudaStream_t st) {
    launch_hi(tg_trig_kernel, dim3(g.p.R), dim3(128), 0, st, g);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}
