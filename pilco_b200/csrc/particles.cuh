// particles.cuh -- what the particle kernels of particles.cu, particles_angles.cu, particles_noise.cu,
// particles_explore.cu, particles_cscore.cu, particles_resample.cu, particles_mlp.cu and particles_features.cu share: the
// per-particle argument structs, the reward value at a point, the step's work at a given state, the fixed-order block
// sum, and the angle, noise, exploration, consistent-score, resampling, MLP-policy and feature-sample kernels' launchers
// (DESIGN.md sections 11, 12, 20, 23, 24, 25, 26, 29 and 30).
#pragma once
#include <initializer_list>
#include "common.cuh"
#include "risk_math.cuh"
#include "trig_math.cuh"

#define PT_THREADS 128
#define PT_MAX_P   (65535 * 32)         // pilco_gp_predict's T limit
#define PT_RBF_VAR 1e-6                 // output variance of the deterministic-GP policy (mode 1, mm_finish_device)
#define PT_INV_PI  0.31830988618379067154

// the policy and the rewards, as every per-particle kernel reads them (pt_policy)
struct PtPolicy {
    int P, H, Ds, U;
    int pol_kind, squash;
    const double* maxa;
    const double* W; const double* b;                   // linear policy [U,Ds], [U]
    const double* C; const double* ell; const double* sf2; const double* beta; int bf;   // RBF policy (bf = 0: linear)
    long long W_bs, b_bs, C_bs, ell_bs, sf2_bs, beta_bs;   // per-restart policy strides (0: shared)
    int n_rewards, n_mult; pilco_reward_term rewards[8]; double mult_mu;
};

struct PtDev : PtPolicy {
    int t;
    const double* x0; const double* eps;                // [P,Ds], [P,H,Ds]: shared by the restarts
    double* traj; double* act; double* step_reward; double* step_risk; double* ret;   // rows r P + p
    double* xt;                                         // predict input [R P,D]
    const double* mean; const double* var;              // predict outputs [R P,Ds]
};

// one reward term at the point x (registers; xg = the same point in global memory, for the box's indexed reads):
// the closed forms of small_kernels.cuh at s = 0
__device__ __forceinline__ double pt_reward_value(const pilco_reward_term& rt, const double (&x)[MAXD], const double* xg,
                                                  int Ds) {
    if (rt.kind == PILCO_REWARD_BOX) return risk_box_point(rt.W, xg);
    if (rt.kind == PILCO_REWARD_LINEAR) {
        double mu = 0.0;
#pragma unroll
        for (int i = 0; i < MAXD; ++i) if (i < Ds) mu = fma(x[i], rt.W[i], mu);
        return mu;
    }
    double v[MAXD];                                     // exp(-0.5 (x-t)' W (x-t)), dev_exp_reward's order
#pragma unroll
    for (int i = 0; i < MAXD; ++i) v[i] = i < Ds ? x[i] - rt.t[i] : 0.0;
    double quad = 0.0;
#pragma unroll
    for (int i = 0; i < MAXD; ++i) {
        if (i < Ds) {
            double wy = 0.0;
#pragma unroll
            for (int k = 0; k < MAXD; ++k) if (k < Ds) wy = fma(rt.W[i * Ds + k], v[k], wy);
            quad = fma(v[i], wy, quad);
        }
    }
    return exp(-0.5 * quad);
}

// pt_step_kernel's work at step t once particle row's state x_t is known (restart r, tr = its traj[:, t] row; DESIGN.md
// section 11): traj[:, t], and for t < H the state terms' reward and risk at x_t, x~_t and the squashed action; at
// t = H the return.  pr_step_kernel (particles_resample.cu) runs it on x_t from the Gaussian refit.  It is a copy of
// pt_step_kernel's code in the same order, kept apart: routing pt_step_kernel through it changes that kernel's register
// allocation, and pt_step_kernel's SASS is pinned.  Keep the two in step.
__device__ __forceinline__ void pt_step_at(const PtDev& a, int r, size_t row, double* tr, const double (&x)[MAXD]) {
    const int Ds = a.Ds, U = a.U, D = Ds + U, t = a.t, H = a.H;
#pragma unroll
    for (int d = 0; d < MAXD; ++d) if (d < Ds) tr[d] = x[d];
    const size_t ph = row * H;
    if (t == H) {                                       // return: step order, as ro_reward_sum_kernel
        double s = 0.0;
        for (int tt = 0; tt < H; ++tt) s += a.step_reward[ph + tt];
        if (a.n_mult > 0) {
            double mult = 1.0;
            for (int tt = 0; tt < H; ++tt) mult *= 1.0 - a.step_risk[ph + tt];
            s += a.mult_mu * (1.0 - mult);
        }
        a.ret[row] = s;
        return;
    }
    double rew = 0.0, risk = 0.0;                       // at the pre-step state (pilco.py:130-134)
    for (int k = 0; k < a.n_rewards; ++k) {
        const pilco_reward_term& rt = a.rewards[k];
        const double v = pt_reward_value(rt, x, tr, Ds);
        if (rt.channel == PILCO_CHANNEL_MULT) risk = fma(rt.coef, v, risk);
        else rew = fma(rt.coef, v, rew);
    }
    a.step_reward[ph + t] = rew;
    a.step_risk[ph + t] = risk;
    double* xo = a.xt + row * D;
#pragma unroll
    for (int d = 0; d < MAXD; ++d) if (d < Ds) xo[d] = x[d];
    double* ao = a.act + (ph + t) * U;
    // squash_sin at a point with the policy's output variance su: maxa exp(-su/2) sin(u)  (dev_squash_sin's form).
    // sin(u) as sinpi(u / pi): its argument reduction is exact, so the kernel carries no Payne-Hanek slow path (whose
    // table lives in local memory); the rounding of u / pi moves the angle by |u| 1.1e-16 at most.
    const double su = a.pol_kind == PILCO_POLICY_RBF ? PT_RBF_VAR : 0.0;
    for (int j = 0; j < U; ++j) {
        double u;
        if (a.pol_kind == PILCO_POLICY_LINEAR) {        // dev_linear_action's order
            const double* W = a.W + r * a.W_bs;
            u = a.b[r * a.b_bs + j];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < Ds) u = fma(W[j * Ds + d], x[d], u);
        } else {                                        // sum_i beta_ji sf2_j exp(-0.5 |(x - c_i) / ell_j|^2)
            const double* ell = a.ell + r * a.ell_bs;
            double il[MAXD];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) il[d] = d < Ds ? 1.0 / ell[j * Ds + d] : 0.0;
            const double sf2 = a.sf2[r * a.sf2_bs + j];
            const double* be = a.beta + r * a.beta_bs + (size_t)j * a.bf;
            const double* C = a.C + r * a.C_bs;
            u = 0.0;
            for (int i = 0; i < a.bf; ++i) {
                const double* c = C + (size_t)i * Ds;
                double d2 = 0.0;
#pragma unroll
                for (int d = 0; d < MAXD; ++d) if (d < Ds) { const double q = (x[d] - c[d]) * il[d]; d2 = fma(q, q, d2); }
                u = fma(sf2 * exp(-0.5 * d2), be[i], u);
            }
        }
        if (a.squash) u = a.maxa[j] * exp(-0.5 * su) * sinpi(u * PT_INV_PI);
        ao[j] = u;
        xo[Ds + j] = u;
    }
}

// fixed-order block sum of NV values per thread (256 threads): warp butterflies, then warps in order -> out[0..NV)
template <int NV>
__device__ __forceinline__ void pg_block_sum(double (&v)[NV], double* red, double* out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int c = 0; c < NV; ++c) {
        const double s = warp_sum(v[c]);
        if (lane == 0) red[c * 8 + warp] = s;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < NV; c += 256) {
        double s = 0.0;
        for (int w = 0; w < 8; ++w) s += red[c * 8 + w];
        out[c] = s;
    }
    __syncthreads();
}

// the reverse sweep's step arguments (pg_step_kernel, particles.cu)
struct PgDev : PtPolicy {
    int t;
    const double* eps; const double* traj; const double* step_risk;
    const double* gxt;          // VJP of step t at x~_t [R P,D]; NULL at t = H-1
    const double* var_prev;     // var_{t-1} [R P,Ds] (t > 0)
    double* gx;                 // [R P,Ds] x_bar_{t+1} in, x_bar_t out (= the gmean of step t-1's VJP)
    double* gvar;               // [R P,Ds] the gvar of step t-1's VJP
    double* zbar;               // [R P,H,U]
};

// ---- angular state dimensions (particles_angles.cu, DESIGN.md section 20) -------------------------------------------
// PtPolicy::Ds is the policy's input width Dh = E + A; x0, eps, traj, mean, var, gx, gvar and var_prev are in the raw
// state width E; x~_t = [phi(x_t), u_t] has D = Dh + U.
struct PaStep : PtDev {
    int E;
    TrigMap tm;                                         // tm.Ds = E
    double* phi;                                        // phi(x_t) [R P,H+1,Dh] for the gradients, or NULL
};

struct PaBwd : PgDev {
    int E;
    TrigMap tm;
    const double* phi;                                  // phi(x_t) [R P,H+1,Dh], the forward's
    double* phib;                                       // phi_bar_t [R P,D] rows (over gxt's; NULL when gxt is)
};

// grid (ceil(P / 128), R): the angle path's forward step t (in place of pt_step_kernel)
int pa_step_launch(cudaStream_t st, dim3 grid, const PaStep& a);
// grid (ceil(P / 128), R): the angle path's reverse step t (in place of pg_step_kernel), two launches
int pa_reverse_launch(cudaStream_t st, dim3 grid, const PaBwd& a);

// ---- measurement noise at the policy's input (particles_noise.cu, DESIGN.md section 23) ------------------------------
// z_t = x_t + sqrt(v) o nu_t; the policy sees phi(z_t), the dynamics GP [phi(x_t), u_t].  Without angles tm is the
// identity map (A = 0).
struct PnNoise {
    const double* nu;                                   // [P,H,E] standard normals, shared by the restarts
    double sv[MAXD];                                    // sqrt(v_i), i < E (0 beyond)
};

struct PnStep : PaStep {
    PnNoise nz;
    double* phiz;                                       // phi(z_t) [R P,H+1,Dh] for the gradients, or NULL
};

struct PnBwd : PaBwd {                                  // phib = NULL: phi_bar_x stays in gxt[:Dh]
    const double* phiz;                                 // phi(z_t) [R P,H+1,Dh], the forward's
    double* phibz;                                      // phi_bar_z,t [R P,Dh] (written when gxt is not NULL)
};

// grid (ceil(P / 128), R): the noisy forward step t (in place of pt_step_kernel / pa_step_kernel)
int pn_step_launch(cudaStream_t st, dim3 grid, const PnStep& a);
// grid (ceil(P / 128), R): the noisy reverse step t (in place of pg_step_kernel / pa_reverse_launch), two launches
int pn_reverse_launch(cudaStream_t st, dim3 grid, const PnBwd& a);

// ---- exploration objective (particles_explore.cu, DESIGN.md section 24) -----------------------------------------------
// Per restart r and step t < H over the restart's P particles, for each ADD-channel term k (K = n_rewards slots; MULT
// slots stay 0): r_kpt at x_pt (state terms, raw) or x~_pt = [phi(x_pt), u_pt] (joint terms), its mean and unbiased
// sample variance, sigma_t^2 = sum_k c_k^2 s_kt^2 and sigma_t = sqrt(sigma_t^2) (0 at or below 1e-12).
struct PxMom {
    int P, H, U, n_rewards;
    TrigMap tm;                                         // tm.Ds = E; the identity map without angles
    const double* traj; const double* act;              // [R P,H+1,E], [R P,H,U]
    pilco_reward_term rewards[8];
    double b;
    double* step_mean; double* step_var;                // [R,H] sum_k c_k mean_kt and sigma_t^2, or NULL
    double* sd;                                         // [R,H] sigma_t, or NULL
    double* tab;                                        // [R,H,K,2] (mean_kt, P b c_k^2 / ((P-1) sigma_t)), or NULL
};

// the bonus's share of step t's reverse step: sum_k a_kpt grad r_k, a_kpt = tab_kt.w (r_kpt - mean_kt)
struct PxBonus {
    int P, H, E, D, t, n_rewards;
    pilco_reward_term rewards[8];
    const double* traj;                                 // [R P,H+1,E]
    const double* xh;                                   // x~_t [R P,D] (the forward's history slot of step t)
    const double* tab;                                  // [R,H,K,2]
    double* gx;                                         // [R P,E] state terms' share
    double* gxt;                                        // [R P,D] joint terms' share
};

// grid (H, R), 256 threads; H = 0 launches nothing
int px_moments_launch(cudaStream_t st, int R, const PxMom& a);
// grid (ceil(P / 128), R)
int px_bonus_launch(cudaStream_t st, dim3 grid, const PxBonus& a);
// value[r] += b sum_t sd[r,t], step order
int px_value_launch(cudaStream_t st, int R, int H, double b, const double* sd, double* value);

// ---- score-function gradient over consistent function samples (particles_cscore.cu, DESIGN.md section 25) ------------
// The whitening reverse of R restarts (T = R P rows, Ds = E): from the consistent forward's packed rows and pivots, eps
// and the weights w_pt = G_pt - (S_t - G_pt) / (P - 1) (P = 1: G_pt), the cotangents of every step's mean' and var'.
struct PcWhite {
    int P, T, H, Ds;
    const double* L;                                    // [H(H+1)/2, E, T] the forward's packed rows
    const double* eps;                                  // [P,H,E], shared by the restarts
    const double* var;                                  // [H,T,E] var'_t = max(d2_t, 0), the forward's history
    const double* G;                                    // [H-1,T] return-to-go (ps_togo_kernel)
    const double* S;                                    // [R,H] its per-(restart, step) sums (ps_base_kernel)
    double* mbar; double* vbar;                         // [H-1,T,E] m_bar_t, v_bar_t
};

// grid (ceil(P / 8), E, R), 256 threads; H < 2 launches nothing
int pc_white_launch(cudaStream_t st, int R, const PcWhite& a);

// ---- Gaussian-resampled particles (particles_resample.cu, DESIGN.md section 26) ----------------------------------------
// At every step t >= 1 restart r's pre-fit particles x'_t (the step closure) are refitted to a Gaussian and redrawn:
// x_pt = mu^_t + L^_t xi_{p,t-1}, mu^_t and S^_t = L^_t L^_t' the sample mean and unbiased covariance of x'_t over the
// restart's P particles (pr_chol's degenerate-column rule).  The step-wise sampler only: Ds = E (no angles).
struct PrFwd {
    int P, H, Ds;
    const double* x0; const double* xi;                 // [P,Ds], [P,H,Ds]: shared by the restarts
    double* xp;                                         // x'_t at slot t-1 of [H,T,Ds]
    double* mu; double* L;                              // mu^_t, L^_t at slot t-1 of [H,R,Ds], [H,R,Ds,Ds]
    double* step_mean; double* step_cov;                // [R,H+1,Ds], [R,H+1,Ds,Ds] (t = 0: x0's moments), or NULL
};

// step a.t of the resampled forward, in place of the step kernel: t = 0 (after pt_step<0>) x0's moments when they are
// asked for; t >= 1 the closure into x'_t, the moments and factor (grid R) and pr_step_kernel, which redraws x_t and
// does pt_step_kernel's work at it.  grid = (ceil(P / 128), R).  net (an MLP policy, DESIGN.md section 29):
// pm_refit_kernel (particles_mlp.cu) in place of pr_step_kernel.
struct PmNet;
int pr_step_launch(cudaStream_t st, dim3 grid, const PtDev& a, const PrFwd& f, const PmNet* net = nullptr);

// the refit's reverse at step t (1 <= t <= H-1), after the reverse step kernel has left y_bar_p = the cotangent of the
// refitted x_pt in gx: gx <- the cotangent of x'_pt, gvar <- that of var_{t-1}
struct PrBwd {
    int P, H, Ds, t;
    const double* xi; const double* eps;                // [P,H,Ds]
    const double* xp; const double* mu; const double* L;   // the forward's histories
    const double* var_prev;                             // var_{t-1} [T,Ds]
    double* gx; double* gvar;                           // [T,Ds]
    double* sc;                                         // [R,Ds+Ds Ds]: mu_bar / P and (A + A') / (P-1)
};

// grid = (ceil(P / 128), R): pr_adjoint_kernel (grid R), then pr_scatter_kernel
int pr_reverse_launch(cudaStream_t st, dim3 grid, const PrBwd& b);

// ---- tanh MLP policies (particles_mlp.cu, DESIGN.md section 29) ---------------------------------------------------------
// h_1 = tanh(A_1 [x; 1]), (L = 2) h_2 = tanh(A_2 [h_1; 1]), z = A_out [h_L; 1]; every A row-major [out, in + 1], the bias
// its last column; theta = the A blocks in that order, restart r's at theta + r theta_bs.  The step kernels read the
// policy from PmNet (PtPolicy's linear and RBF fields are unused); everything else is the linear path's.
#define PM_MAXW   64                    // widest hidden layer
#define PM_CHUNKS 16                    // the reduction's particle chunks per restart (at most)
struct PmNet {
    int L, w1, w2;                      // w2 = 0 when L = 1
    int n_theta, off2, offo;            // theta's length; where A_2 (L = 2) and A_out start
    const double* theta; long long theta_bs;
};

// The reverse step's per-particle buffers, feature-major [width, RPp] (column row = r Pp + p; Pp = the restart's rows
// padded to whole reduction chunks, the padding zero): the layer inputs [x; 1], [h_1; 1], [h_2; 1] and the
// pre-activation cotangents d_1, d_2, d_out (= z_bar_t) of the current step
struct PmBwd {
    PmNet net;
    long long RPp, Pp;
    double* in0; double* in1; double* in2;
    double* d1; double* d2; double* dout;
};

// grid (ceil(P / 128), R): the MLP's forward step t, in place of pt_step_kernel
int pm_step_launch(cudaStream_t st, dim3 grid, const PtDev& a, const PmNet& m);
// grid (ceil(P / 128), R): the MLP's refit step t >= 1, in place of pr_step_kernel
int pm_refit_launch(cudaStream_t st, dim3 grid, const PtDev& a, const PrFwd& f, const PmNet& m);
// grid (ceil(P / 128), R): the MLP's reverse step t, in place of pg_step_kernel (x_bar_t, var_bar_{t-1}; with a.gxt the
// step's layer inputs and cotangents into b's buffers)
int pm_reverse_launch(cudaStream_t st, dim3 grid, const PgDev& a, const PmBwd& b);
// gtheta [R, n_theta] = (1/P) sum of the chunk partials part [R, nc, n_theta] in chunk order; value [R] = the mean return
int pm_finish_launch(cudaStream_t st, int R, int P, int nc, int n_theta, const double* part, const double* ret,
                     double* gtheta, double* value);

// ---- function samples from random-feature draws (particles_features.cu, DESIGN.md section 30) -------------------------
// f_pe(x~) = phi_e(x~)' w_pe + sum_j sf2_e exp(-0.5 |(x~ - X_j) / ell_e|^2) v_pe,j at the T = R P rows of x~ (row r P + p
// reads particle p's draws: the restarts share them)
struct PfDev {
    long long T;
    int P, D, E, F, n;
    const double* omega;                                // [E,F,D]
    const double* X; const double* ell; const double* sf2;   // the dynamics GP's [n,D], [E,D], [E]
    const double* w; const double* v;                   // [P,E,2F], [P,E,n]
    const double* xh;                                   // x~_t [T,D]
    double* mean; double* var;                          // [T,E] eval: f and 0
    const double* gmean;                                // [T,E] VJP: m_bar
    double* gxt;                                        // [T,D] VJP: x~_bar
};

// grid (ceil(T / 8), E): mean = f(x~_t), var = 0
int pf_eval_launch(cudaStream_t st, const PfDev& a);
// grid ceil(T / 8): gxt = sum_e gmean_e d f_e / d x~ at x~_t
int pf_vjp_launch(cudaStream_t st, const PfDev& a);
