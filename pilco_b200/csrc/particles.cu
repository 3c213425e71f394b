// particles.cu -- Monte Carlo particle rollout of the learnt dynamics under the policy (fp64):
//   pilco_particles_rollout   P particles x H steps of the Markov chain whose Gaussian marginals the moment-matching
//                             cascade (rollout.cu) approximates; the caller supplies x0 and the standard normals
//   u_t = squash(pi(x_t)),  x_{t+1} = x_t + mu(x~_t) + sqrt(max(var(x~_t), 0)) o eps_t,  x~_t = [x_t, u_t]
// Launch sequence (one stream, graph-capturable, no host sync; DESIGN.md section 11):
//   pt_step<0>, predict, pt_step<1>, predict, ..., predict, pt_step<H>
// pt_step_kernel is one thread per particle: it closes the previous step from the predict outputs, writes traj[:, t],
// and for t < H evaluates the reward terms at the point x_t, the policy and the predict input x~_t; at t = H it sums
// the return.  The O(n^2) work per step is pilco_gp_predict (predict.cu) at T = P.
// pilco_particles_rollout_batch_grad runs R policies over the same x0 and eps (DESIGN.md section 13): restart r is
// blockIdx.y of the per-particle kernels, its particle p is row r P + p of every output and of the predict calls
// (T = R P), and its policy arrays are offset by r times their batch strides.  The unbatched entry points are the
// same launches at R = 1.
// pilco_particles_rollout_consistent draws ONE posterior function per particle (DESIGN.md section 14): after each step's
// predict (fs_predict_kernel, predict.cu, which also keeps W_t = K*_t iK and K*_t) fs_cond_kernel conditions the draw
// on the particle's earlier inputs, and pt_step_kernel closes the step unchanged from the mean and variance it leaves.
// pilco_particles_rollout_score_grad runs the batched forward and then the score-function gradient (DESIGN.md section
// 16): per-transition weights and score cotangents, one VJP pass over all steps, z_bar, and the pathwise reduction.
// Joint state-action reward terms (PILCO_REWARD_*_SA, DESIGN.md section 18) have kernels of their own, launched beside
// the per-particle ones only when such a term is present: pt_joint_kernel adds their values at x~_t to the step's
// reward and risk after pt_step<t>, pj_grad_kernel adds their gradients to the VJP output x~_bar_t before pg_step<t> /
// ps_zbar.  The state kernels see the state terms only (pt_policy), so they are untouched: pt_step_kernel and
// pg_step_kernel sit at their register limits (127 and 255), and the joint terms would have spilled them.
// Angular state dimensions (pilco_particles_angles_*, DESIGN.md section 20): pt_forward, pg_reverse and ps_run take the
// angles' map and launch the step kernels of particles_angles.cu in place of pt_step / pg_step; the shared structs are
// in particles.cuh.
// Measurement noise at the policy's input (pilco_particles_noisy_*, DESIGN.md section 23): the same drivers take a
// PnNoise next to the map (the identity map without angles) and launch the kernels of particles_noise.cu in place of the
// angle step kernels; the policy inputs of the reductions are then the phi(z) history.
// The exploration objective (pilco_particles_explore_*, DESIGN.md section 24): pt_call launches the kernels of
// particles_explore.cu beside the others (the moments after the forward, the bonus's share before each reverse step
// kernel, the bonus into value after the reduction).
// Gaussian-resampled particles (pilco_particles_resampled_*, DESIGN.md section 26): pt_forward launches
// pr_step_launch's kernels (particles_resample.cu) in place of pt_step<t> for t >= 1, and pg_reverse the refit's reverse
// stage after the step kernel of each t = H-1 .. 1.
// The score-function gradient over consistent function samples (pilco_particles_consistent_score_grad_*, DESIGN.md
// section 25): ps_run on the consistent forward; pc_white_kernel (particles_cscore.cu) turns the weights into the
// cotangents of every step's mean' and var', which the reverse of the conditioning and the predict VJP carry to
// x~_bar_t step by step.
// Time-varying linear policies (pilco_particles_scheduled_*, DESIGN.md section 28): pt_forward and pg_reverse hand step
// t's launches W + t W_ts and b + t b_ts; ps_zbar_sched_kernel and pg_sched_kernel stand in for the two kernels that
// cover all H steps in one grid (ps_zbar_kernel, pg_param_kernel).
// Tanh MLP policies (pilco_particles_mlp_*, DESIGN.md section 29): pt_forward launches the step kernels of
// particles_mlp.cu in place of pt_step / pr_step, pg_reverse its reverse step kernel in place of pg_step followed by one
// batched gemm() per layer (factorize.cu) into per-chunk partials, and pm_finish_kernel in place of pg_reduce.
// Function samples from random-feature draws (pilco_particles_features_* and _mlp_features_*, DESIGN.md section 30):
// pt_forward launches pf_eval_kernel (particles_features.cu) in place of the predict, which leaves mean = f(x~_t) and
// var = 0 for the unchanged step kernels, and pg_reverse pf_vjp_kernel in place of the predict VJP.
#include <cmath>
#include "particles.cuh"
#include "gemm.cuh"

// grid (ceil(P / 128), R), one thread per particle p of restart r = blockIdx.y
__global__ void __launch_bounds__(PT_THREADS) pt_step_kernel(PtDev a) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= a.P) return;
    const int Ds = a.Ds, U = a.U, D = Ds + U, t = a.t, H = a.H;
    const size_t row = (size_t)r * a.P + p;
    double* tr = a.traj + (row * (H + 1) + t) * Ds;
    double x[MAXD];
    if (t == 0) {
#pragma unroll
        for (int d = 0; d < MAXD; ++d) x[d] = d < Ds ? a.x0[(size_t)p * Ds + d] : 0.0;
    } else {                                            // close step t-1
        const double* xp = tr - Ds;
        const double* mu = a.mean + row * Ds;
        const double* var = a.var + row * Ds;
        const double* ep = a.eps + ((size_t)p * H + (t - 1)) * Ds;
#pragma unroll
        for (int d = 0; d < MAXD; ++d) {
            if (d < Ds) {
                const double v = var[d];
                x[d] = fma(sqrt(v < 0.0 ? 0.0 : v), ep[d], xp[d] + mu[d]);      // NaN stays NaN
            } else x[d] = 0.0;
        }
    }
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

// ---- joint state-action reward terms (DESIGN.md section 18) --------------------------------------------------------
// rewards[] = the joint terms only; n_mult counts the MULT terms of both kinds.  Buffers have T = R P rows.
struct PjDev : PtPolicy {
    long long T;
    int t;                                              // pt_joint: the step; pj_grad: the first step of the grid
    const double* xh;                                   // pt_joint: x~_t [T,D]; pj_grad: x~ of every step [H,T,D]
    double* step_reward; double* step_risk;             // [T,H]
    double* gxt; long long gstep;                       // x~_bar of step t at gxt + t gstep (0: one [T,D] buffer)
    int first;                                          // first dimension of x~_bar that receives (0, or Ds: actions only)
};

// exp(-0.5 v' W v), v = x~ - t, or x~' W, at the point xq [D] in global memory: plain loops, a handful of registers
__device__ __forceinline__ double pj_value(const pilco_reward_term& rt, const double* xq, int D) {
    double acc = 0.0;
    if (rt.kind == PILCO_REWARD_LINEAR_SA) {
        for (int i = 0; i < D; ++i) acc = fma(xq[i], rt.W[i], acc);
        return acc;
    }
    for (int i = 0; i < D; ++i) {
        double wy = 0.0;
        for (int k = 0; k < D; ++k) wy = fma(rt.W[i * D + k], xq[k] - rt.t[k], wy);
        acc = fma(xq[i] - rt.t[i], wy, acc);
    }
    return exp(-0.5 * acc);
}

// grid (ceil(P / 128), R), one thread per particle p of restart r = blockIdx.y, after pt_step<t>: the joint terms at
// x~_t join the step's reward and risk (state terms first, then these, each in term order)
__global__ void __launch_bounds__(PT_THREADS) pt_joint_kernel(PjDev a) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x;
    if (p >= a.P) return;
    const int D = a.Ds + a.U;
    const size_t row = (size_t)blockIdx.y * a.P + p, o = row * a.H + a.t;
    const double* xq = a.xh + row * D;
    double rew = a.step_reward[o], risk = a.step_risk[o];
    for (int k = 0; k < a.n_rewards; ++k) {
        const pilco_reward_term& rt = a.rewards[k];
        const double v = pj_value(rt, xq, D);
        if (rt.channel == PILCO_CHANNEL_MULT) risk = fma(rt.coef, v, risk);
        else rew = fma(rt.coef, v, rew);
    }
    a.step_reward[o] = rew;
    a.step_risk[o] = risk;
}

// grid (ceil(P / 128) nsteps, R), one thread per (step t = a.t + blockIdx.x / nb, particle p of restart r = blockIdx.y):
// x~_bar_t[first:] += sum_k a_kt grad v_k(x~_t), a_kt as in the reverse sweep below (coef_k, or coef_k mult_mu
// prod_{s != t} (1 - risk_s) in the MULT channel)
__global__ void __launch_bounds__(PT_THREADS) pj_grad_kernel(PjDev a) {
    PDL_ENTRY();
    const int nb = (a.P + PT_THREADS - 1) / PT_THREADS;
    const int t = a.t + blockIdx.x / nb, p = (blockIdx.x % nb) * PT_THREADS + threadIdx.x;
    if (p >= a.P) return;
    const int D = a.Ds + a.U, H = a.H;
    const size_t row = (size_t)blockIdx.y * a.P + p;
    const double* xq = a.xh + ((size_t)t * a.T + row) * D;
    double* g = a.gxt + (size_t)t * a.gstep + row * D;
    double wmult = 0.0;
    if (a.n_mult > 0) {                                 // as pg_step_kernel
        const double* rk = a.step_risk + row * H;
        double pre = 1.0, suf = 1.0;
        for (int s = 0; s < t; ++s) pre *= 1.0 - rk[s];
        for (int s = t + 1; s < H; ++s) suf *= 1.0 - rk[s];
        wmult = a.mult_mu * (pre * suf);
    }
    for (int k = 0; k < a.n_rewards; ++k) {
        const pilco_reward_term& rt = a.rewards[k];
        const double w = rt.channel == PILCO_CHANNEL_MULT ? rt.coef * wmult : rt.coef;
        if (rt.kind == PILCO_REWARD_LINEAR_SA) {
            for (int i = a.first; i < D; ++i) g[i] = fma(w, rt.W[i], g[i]);
            continue;
        }
        const double f = -0.5 * w * pj_value(rt, xq, D);        // gradient -value (W + W') v / 2
        for (int i = a.first; i < D; ++i) {
            double wv = 0.0;
            for (int k2 = 0; k2 < D; ++k2) wv = fma(rt.W[i * D + k2] + rt.W[k2 * D + i], xq[k2] - rt.t[k2], wv);
            g[i] = fma(f, wv, g[i]);
        }
    }
}

// ---- reverse sweep of pilco_particles_rollout_grad (DESIGN.md section 12) ---------------------------------------------
// Per particle, x_bar_H = 0 and t = H-1 .. 0 (s_t = sqrt(max(var_t, 0)), z_t the pre-squash action):
//   mu_bar_t = x_bar_{t+1},  var_bar_t = x_bar_{t+1} o eps_t / (2 s_t) where var_t > 0, else 0
//   x~_bar_t = pilco_gp_predict_vjp at x~_t;  z_bar_t = x~_bar_t[Ds:] o maxa e^{-su/2} cos(z_t)  (when squashed)
//   x_bar_t  = x_bar_{t+1} + x~_bar_t[:Ds] + (d pi / dx)' z_bar_t + sum_k a_kt grad v_k(x_t)
// a_kt = coef_k (ADD) or coef_k mult_mu prod_{s != t} (1 - risk_s) (MULT).  x_H carries no reward, so the sweep
// starts at t = H-1 with x_bar_H = 0 and x~_bar_{H-1} = 0: H-1 VJP calls.  With joint terms pj_grad_kernel has added
// sum_k a_kt grad v_k(x~_t) to x~_bar_t beforehand (at t = H-1 to a zeroed one, which this kernel then reads).
// Its arguments: PgDev (particles.cuh).

// grid (ceil(P / 128), R), one thread per particle p of restart r = blockIdx.y: step t of the reverse sweep
__global__ void __launch_bounds__(PT_THREADS) pg_step_kernel(PgDev a) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= a.P) return;
    const int Ds = a.Ds, U = a.U, t = a.t, H = a.H;
    const size_t row = (size_t)r * a.P + p;
    const double* xg = a.traj + (row * (H + 1) + t) * Ds;
    const double* gxt = a.gxt ? a.gxt + row * (Ds + U) : nullptr;
    double x[MAXD], xb[MAXD];
#pragma unroll
    for (int d = 0; d < MAXD; ++d) {
        x[d] = d < Ds ? xg[d] : 0.0;
        xb[d] = (d < Ds && gxt) ? a.gx[row * Ds + d] + gxt[d] : 0.0;
    }
    // reward terms at x_t (box: flat almost everywhere, no gradient)
    double wmult = 0.0;
    if (a.n_mult > 0) {                                 // mult_mu prod_{s != t} (1 - risk_s): prefix x suffix, no division
        const double* rk = a.step_risk + row * H;
        double pre = 1.0, suf = 1.0;
        for (int s = 0; s < t; ++s) pre *= 1.0 - rk[s];
        for (int s = t + 1; s < H; ++s) suf *= 1.0 - rk[s];
        wmult = a.mult_mu * (pre * suf);
    }
    for (int k = 0; k < a.n_rewards; ++k) {
        const pilco_reward_term& rt = a.rewards[k];
        if (rt.kind == PILCO_REWARD_BOX) continue;
        const double w = rt.channel == PILCO_CHANNEL_MULT ? rt.coef * wmult : rt.coef;
        if (rt.kind == PILCO_REWARD_LINEAR) {
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < Ds) xb[d] = fma(w, rt.W[d], xb[d]);
            continue;
        }
        // exp(-0.5 v' W v), v = x - t:  gradient -value (W + W') v / 2
        double v[MAXD], gv[MAXD];
#pragma unroll
        for (int i = 0; i < MAXD; ++i) v[i] = i < Ds ? x[i] - rt.t[i] : 0.0;
        double quad = 0.0;
#pragma unroll
        for (int i = 0; i < MAXD; ++i) {
            gv[i] = 0.0;
            if (i < Ds) {
                double wy = 0.0, wty = 0.0;
#pragma unroll
                for (int k2 = 0; k2 < MAXD; ++k2)
                    if (k2 < Ds) { wy = fma(rt.W[i * Ds + k2], v[k2], wy); wty = fma(rt.W[k2 * Ds + i], v[k2], wty); }
                quad = fma(v[i], wy, quad);
                gv[i] = wy + wty;
            }
        }
        const double f = -0.5 * w * exp(-0.5 * quad);
#pragma unroll
        for (int d = 0; d < MAXD; ++d) if (d < Ds) xb[d] = fma(f, gv[d], xb[d]);
    }
    // policy: z_bar_t and (d pi / dx)' z_bar_t; z_t recomputed in the forward's order.  This is pt_step_kernel's
    // policy code with the Jacobian row added: one shared function changes pt_step_kernel's code (127 -> 96 registers)
    // and makes the rollout slower at small P, so the two stay separate and must be kept in the same order.
    double* zb = a.zbar + (row * H + t) * U;
    const double su = a.pol_kind == PILCO_POLICY_RBF ? PT_RBF_VAR : 0.0;
    for (int j = 0; j < U; ++j) {
        if (!gxt) { zb[j] = 0.0; continue; }
        double jx[MAXD], z;
        if (a.pol_kind == PILCO_POLICY_LINEAR) {
            const double* W = a.W + r * a.W_bs;
            z = a.b[r * a.b_bs + j];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) {
                jx[d] = d < Ds ? W[j * Ds + d] : 0.0;
                if (d < Ds) z = fma(W[j * Ds + d], x[d], z);
            }
        } else {                                        // d z_j / dx = sum_i beta_ji k_ji (c_i - x) / ell_j^2
            const double* ell = a.ell + r * a.ell_bs;
            double il[MAXD];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) { il[d] = d < Ds ? 1.0 / ell[j * Ds + d] : 0.0; jx[d] = 0.0; }
            const double sf2 = a.sf2[r * a.sf2_bs + j];
            const double* be = a.beta + r * a.beta_bs + (size_t)j * a.bf;
            const double* C = a.C + r * a.C_bs;
            z = 0.0;
            for (int i = 0; i < a.bf; ++i) {
                const double* c = C + (size_t)i * Ds;
                double d2 = 0.0;
#pragma unroll
                for (int d = 0; d < MAXD; ++d) if (d < Ds) { const double q = (x[d] - c[d]) * il[d]; d2 = fma(q, q, d2); }
                const double kb = sf2 * exp(-0.5 * d2);
                z = fma(kb, be[i], z);
                const double f = kb * be[i];
#pragma unroll
                for (int d = 0; d < MAXD; ++d) if (d < Ds) jx[d] = fma(f, (c[d] - x[d]) * (il[d] * il[d]), jx[d]);
            }
        }
        double zbj = gxt[Ds + j];
        // cos(z) as cospi(z / pi): no Payne-Hanek slow path (and its local-memory table), as the forward's sinpi
        if (a.squash) zbj *= a.maxa[j] * exp(-0.5 * su) * cospi(z * PT_INV_PI);
        zb[j] = zbj;
#pragma unroll
        for (int d = 0; d < MAXD; ++d) if (d < Ds) xb[d] = fma(zbj, jx[d], xb[d]);
    }
#pragma unroll
    for (int d = 0; d < MAXD; ++d) if (d < Ds) a.gx[row * Ds + d] = xb[d];
    if (t > 0) {                                        // cotangents of step t-1's predict outputs
        const double* vp = a.var_prev + row * Ds;
        const double* ep = a.eps + ((size_t)p * H + (t - 1)) * Ds;
#pragma unroll
        for (int d = 0; d < MAXD; ++d) {
            if (d < Ds) {
                const double v = vp[d];
                a.gvar[row * Ds + d] = v > 0.0 ? xb[d] * ep[d] / (2.0 * sqrt(v)) : 0.0;
            }
        }
    }
}

struct PgRed : PtPolicy {
    const double* traj; const double* zbar; const double* ret;
    double* gW; double* gb;                             // linear [R,U,Ds], [R,U]
    double* s1; double* s2; double* gbeta;              // RBF per (r, output j, centre i): [R,U,bf,Ds] (x2), [R,U,bf]
    double* gXc; double* gell;                          // RBF direct terms (pg_rbf_finish_kernel) [R,bf,Ds], [R,U,Ds]
    double* value;                                      // [R]
};

// The policy-parameter gradient over all P H points (x_t, z_bar_t) of restart r = blockIdx.y and its value, each CTA
// one fixed-order sum: grid ((linear: U, RBF: U bf) + 1, R), 256 threads; thread q takes the points q, q + 256, ...
// of the restart in order (so a restart's sums do not depend on R).
//   linear j:    gW[j] = sum z_bar_j x / P,  gb[j] = sum z_bar_j / P
//   RBF (j, i):  a = z_bar_j beta_ji k_ji:  s1 = sum a (x - c_i),  s2 = sum a (x - c_i)^2,  gbeta_ji = sum z_bar_j k_ji / P
__global__ void __launch_bounds__(256) pg_param_kernel(PgRed a) {
    PDL_ENTRY();
    __shared__ double red[(2 * MAXD + 1) * 8], out[2 * MAXD + 1];
    const int Ds = a.Ds, U = a.U, H = a.H, tid = threadIdx.x, r = blockIdx.y;
    const size_t npts = (size_t)a.P * H, r0 = (size_t)r * a.P;       // r0: the restart's first row
    const double* traj = a.traj + r0 * (H + 1) * Ds;
    const double* zbar = a.zbar + r0 * H * U;
    const int nblk = a.pol_kind == PILCO_POLICY_LINEAR ? U : U * a.bf;
    const double invP = 1.0 / a.P;
    if ((int)blockIdx.x == nblk) {                      // value = mean return
        double v[1] = {0.0};
        for (int p = tid; p < a.P; p += 256) v[0] += a.ret[r0 + p];
        pg_block_sum<1>(v, red, out);
        if (tid == 0) a.value[r] = out[0] * invP;
        return;
    }
    if (a.pol_kind == PILCO_POLICY_LINEAR) {
        const int j = blockIdx.x;
        double v[MAXD + 1];
#pragma unroll
        for (int d = 0; d <= MAXD; ++d) v[d] = 0.0;
        for (size_t q = tid; q < npts; q += 256) {
            const size_t p = q / H, t = q % H;
            const double* x = traj + (p * (H + 1) + t) * Ds;
            const double zb = zbar[q * U + j];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < Ds) v[d] = fma(zb, x[d], v[d]);
            v[MAXD] += zb;
        }
        pg_block_sum<MAXD + 1>(v, red, out);
        if (tid < Ds) a.gW[((size_t)r * U + j) * Ds + tid] = out[tid] * invP;
        if (tid == 0) a.gb[(size_t)r * U + j] = out[MAXD] * invP;
        return;
    }
    const int j = blockIdx.x / a.bf, i = blockIdx.x % a.bf;
    const double* C = a.C + r * a.C_bs;
    const double* ell = a.ell + r * a.ell_bs;
    double c[MAXD], il[MAXD], v[2 * MAXD + 1];
#pragma unroll
    for (int d = 0; d < MAXD; ++d) {
        c[d] = d < Ds ? C[(size_t)i * Ds + d] : 0.0;
        il[d] = d < Ds ? 1.0 / ell[j * Ds + d] : 0.0;
    }
#pragma unroll
    for (int k = 0; k <= 2 * MAXD; ++k) v[k] = 0.0;
    const double sf2 = a.sf2[r * a.sf2_bs + j], bji = a.beta[r * a.beta_bs + (size_t)j * a.bf + i];
    for (size_t q = tid; q < npts; q += 256) {
        const size_t p = q / H, t = q % H;
        const double* x = traj + (p * (H + 1) + t) * Ds;
        const double zb = zbar[q * U + j];
        double df[MAXD], d2 = 0.0;
#pragma unroll
        for (int d = 0; d < MAXD; ++d) {
            df[d] = d < Ds ? x[d] - c[d] : 0.0;
            const double s = df[d] * il[d];
            d2 = fma(s, s, d2);
        }
        const double k = sf2 * exp(-0.5 * d2), w = zb * bji * k;
        v[2 * MAXD] = fma(zb, k, v[2 * MAXD]);
#pragma unroll
        for (int d = 0; d < MAXD; ++d) { v[d] = fma(w, df[d], v[d]); v[MAXD + d] = fma(w * df[d], df[d], v[MAXD + d]); }
    }
    pg_block_sum<2 * MAXD + 1>(v, red, out);
    const size_t ji = ((size_t)r * U + j) * a.bf + i;
    if (tid < Ds) { a.s1[ji * Ds + tid] = out[tid]; a.s2[ji * Ds + tid] = out[MAXD + tid]; }
    if (tid == 0) a.gbeta[ji] = out[2 * MAXD] * invP;
}

// direct RBF gradients from the per-(j, i) sums, in fixed order; one CTA per restart r = blockIdx.x:
//   gXc[i,d] = sum_j s1[j,i,d] / ell_jd^2 / P,   gell[j,d] = sum_i s2[j,i,d] / ell_jd^3 / P
__global__ void __launch_bounds__(128) pg_rbf_finish_kernel(PgRed a) {
    PDL_ENTRY();
    const int Ds = a.Ds, U = a.U, bf = a.bf, r = blockIdx.x;
    const double invP = 1.0 / a.P;
    const size_t rU = (size_t)r * U;                    // restart r's first (output, centre) block
    for (int q = threadIdx.x; q < bf * Ds; q += 128) {
        const int i = q / Ds, d = q % Ds;
        double s = 0.0;
        for (int j = 0; j < U; ++j) {
            const double l = a.ell[r * a.ell_bs + j * Ds + d];
            s += a.s1[((rU + j) * bf + i) * Ds + d] / (l * l);
        }
        a.gXc[(size_t)r * bf * Ds + q] = s * invP;
    }
    for (int q = threadIdx.x; q < U * Ds; q += 128) {
        const int j = q / Ds, d = q % Ds;
        double s = 0.0;
        for (int i = 0; i < bf; ++i) s += a.s2[((rU + j) * bf + i) * Ds + d];
        const double l = a.ell[r * a.ell_bs + q];
        a.gell[rU * Ds + q] = s / (l * l * l) * invP;
    }
}

// ---- consistent function samples (pilco_particles_rollout_consistent, DESIGN.md section 14) ------------------------
// Particle p follows x_{t+1} = x_t + f(x~_t) with ONE draw f per particle and output from the latent posterior
// k_post(a, b) = k_e(a, b) - k(a, C) iK_e k(C, b), sampled sequentially (exact for a GP with path-dependent inputs):
//   c_s  = k_post(x~_t, x~_s), s < t;   l = L_{<t}^-1 c;   d2 = var(x~_t) - sum_s l_s^2
//   f_t  = mu(x~_t) + sum_{s<t} l_s eps_s + sqrt(max(d2, 0)) eps_t
// A pivot with d2 <= FS_TAU sf2_e (conditional sd below 1e-5 sigma_f: no visible randomness, and d2 in the rounding
// noise of var) leaves its column out of every later substitution: the semidefinite Cholesky, so a revisited input
// reproduces its earlier value.  The step's own noise is sqrt(max(d2, 0)) in every case.
#define FS_TAU   1e-10
#define FS_WARPS 8                      // warps (particles) per CTA of fs_cond_kernel

// Buffers have T = R P rows (restart r's particle p is row r P + p, as section 13); eps is shared by the restarts.
struct FsCond {
    int P, T, H, D, Ds, n, np, t;
    const double* ell; const double* sf2;               // dynamics [E,D], [E]
    const double* xh;                                   // [H,T,D] predict inputs of the steps so far
    const double* mu; const double* s2;                 // [T,Ds] the posterior mean and variance at x~_t
    const double* W;                                    // [E,T,np] W_t = K*_t iK
    const double* Kh;                                   // [H,E,T,np] K*_s of every step
    const double* eps;                                  // [P,H,Ds]
    double* L;                                          // [H(H+1)/2, E, T] packed rows; (s, r) at s(s+1)/2 + r
    double* mean; double* var;                          // [T,Ds] what pt_step_kernel closes the step with
};

__device__ __forceinline__ double fs_bfly(double v) {   // fixed butterfly: every lane ends with the same bits
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// grid (ceil(P / FS_WARPS), E, R), one warp per (particle p of restart r = blockIdx.z, output e): step t's conditioning
// on the particle's past.  The packed diagonal holds the pivot later substitutions divide by: sqrt(d2), or 0 for a
// degenerate column.
__global__ void __launch_bounds__(FS_WARPS * 32, 4) fs_cond_kernel(FsCond a) {
    PDL_ENTRY();
    const int lane = threadIdx.x & 31, p = blockIdx.x * FS_WARPS + (threadIdx.x >> 5), e = blockIdx.y;
    if (p >= a.P) return;
    const int D = a.D, Ds = a.Ds, t = a.t, n = a.n;
    const size_t T = a.T, row = (size_t)blockIdx.z * a.P + p, EP = (size_t)Ds * T, pe = (size_t)e * T + row;
    const double sf2 = a.sf2[e];
    // lane d < D holds dimension d of x~_t and 1 / ell_ed
    const bool dl = lane < D;
    const double xd = dl ? a.xh[((size_t)t * T + row) * D + lane] : 0.0;
    const double ild = dl ? 1.0 / a.ell[(size_t)e * D + lane] : 0.0;
    double* Lt = a.L + (size_t)t * (t + 1) / 2 * EP + pe;              // row t: entry s at Lt[s EP]
    const double* __restrict__ Wr = a.W + pe * a.np;
    // c_s = k_e(x~_t, x~_s) - W_t . K*_s: lanes stride the columns (and the dimensions) in order, then the butterfly
    for (int s = 0; s < t; ++s) {
        const double* __restrict__ Kr = a.Kh + ((size_t)s * EP + pe) * a.np;
        double dot = 0.0;
#pragma unroll 4
        for (int j = lane; j < n; j += 32) dot = fma(Wr[j], Kr[j], dot);
        const double q = dl ? (xd - a.xh[((size_t)s * T + row) * D + lane]) * ild : 0.0;
        dot = fs_bfly(dot);
        const double d2 = fs_bfly(q * q);
        const double c = sf2 * exp(-0.5 * d2) - dot;
        if (lane == 0) Lt[(size_t)s * EP] = c;
    }
    __syncwarp();
    // forward substitution in the particle's running factor, in place: Lt[s] = c_s -> l_s
    for (int s = 0; s < t; ++s) {
        const double* Ls = a.L + (size_t)s * (s + 1) / 2 * EP + pe;
        double sub = 0.0;
        for (int r = lane; r < s; r += 32) sub = fma(Ls[(size_t)r * EP], Lt[(size_t)r * EP], sub);
        sub = fs_bfly(sub);
        const double piv = Ls[(size_t)s * EP];
        const double l = piv > 0.0 ? (Lt[(size_t)s * EP] - sub) / piv : 0.0;
        __syncwarp();                                   // every lane has read c_s before it is overwritten
        if (lane == 0) Lt[(size_t)s * EP] = l;
        __syncwarp();
    }
    double ssq = 0.0, sme = 0.0;
    const double* ep = a.eps + (size_t)p * a.H * Ds + e;
    for (int s = lane; s < t; s += 32) {
        const double l = Lt[(size_t)s * EP];
        ssq = fma(l, l, ssq);
        sme = fma(l, ep[(size_t)s * Ds], sme);
    }
    ssq = fs_bfly(ssq);
    sme = fs_bfly(sme);
    if (lane == 0) {
        const size_t o = row * Ds + e;
        const double mu = a.mu[o], d2 = a.s2[o] - ssq;
        Lt[(size_t)t * EP] = d2 > FS_TAU * sf2 ? sqrt(d2) : 0.0;
        a.mean[o] = t > 0 ? mu + sme : mu;              // t = 0: the marginal sampler's step exactly
        a.var[o] = d2 < 0.0 ? 0.0 : d2;                 // NaN stays NaN
    }
}

// ---- reverse of the conditioning (pilco_particles_rollout_consistent_grad, DESIGN.md section 15) -------------------
// Per (particle, output) at reverse step t, given m_bar = the cotangent of mean'_t and v_bar = that of var'_t, with the
// packed cotangent rows G (Lambda of the factor rows, accumulated by the later steps; zero at the start):
//   d2_bar = piv_t > 0 ? v_bar + Lambda_tt / (2 piv_t) : 0         (tau rule: a degenerate step's own noise is constant)
//   l_bar_s = Lambda_ts + m_bar eps_s - 2 d2_bar l_ts
//   s = t-1 .. 0:  c_s = l_bar_s / piv_s (0 where piv_s = 0);  Lambda_ss -= c_s l_ts;
//                  r < s:  l_bar_r -= c_s l_sr,  Lambda_sr -= c_s l_tr
// Row t of G then holds c_t. = G_t., the cotangent of the cross-covariance k_post(x~_t, x~_s); the entries s > t are in
// rows s (written by the earlier reverse steps).  Out: a_t = -2 d2_bar K*_t - sum_{s != t} G_ts K*_s and the direct
// sum sum_{s != t} G_ts k_e(x~_t, x~_s) (x~_s - x~_t), for fs_predict_vjp_kernel.
struct FsBwd {
    int P, T, H, D, Ds, np, t;
    const double* ell; const double* sf2;               // dynamics [E,D], [E]
    const double* xh;                                   // [H,T,D] predict inputs of every step
    const double* Kh;                                   // [H,E,T,np] K*_s of every step
    const double* L;                                    // [H(H+1)/2, E, T] the forward's packed rows
    const double* eps;                                  // [P,H,Ds]
    const double* gx; const double* gvar;               // [T,Ds] m_bar_t, v_bar_t
    double* G;                                          // [H(H+1)/2, E, T] Lambda, then c (one buffer)
    double* A;                                          // [E,T,np] a_t
    double* dir;                                        // [E,T,D] the direct sums
};

// grid (ceil(P / FS_WARPS), E, R), one warp per (particle p of restart r = blockIdx.z, output e), as fs_cond_kernel
__global__ void __launch_bounds__(FS_WARPS * 32, 3) fs_cond_bwd_kernel(FsBwd a) {
    PDL_ENTRY();
    const int lane = threadIdx.x & 31, p = blockIdx.x * FS_WARPS + (threadIdx.x >> 5), e = blockIdx.y;
    if (p >= a.P) return;
    const int D = a.D, Ds = a.Ds, t = a.t, H = a.H, np = a.np;
    const size_t T = a.T, row = (size_t)blockIdx.z * a.P + p, EP = (size_t)Ds * T, pe = (size_t)e * T + row;
    const double* Lt = a.L + (size_t)t * (t + 1) / 2 * EP + pe;        // row t: entry s at [s EP]
    double* Gt = a.G + (size_t)t * (t + 1) / 2 * EP + pe;
    const double piv = Lt[(size_t)t * EP];
    const size_t o = row * Ds + e;
    const double mb = a.gx[o];
    const double db = piv > 0.0 ? a.gvar[o] + Gt[(size_t)t * EP] / (2.0 * piv) : 0.0;
    const double* ep = a.eps + (size_t)p * H * Ds + e;
    for (int s = lane; s < t; s += 32)
        Gt[(size_t)s * EP] = fma(-2.0 * db, Lt[(size_t)s * EP], fma(mb, ep[(size_t)s * Ds], Gt[(size_t)s * EP]));
    __syncwarp();
    // reverse of the forward substitution, s = t-1 .. 0
    for (int s = t - 1; s >= 0; --s) {
        const double* Ls = a.L + (size_t)s * (s + 1) / 2 * EP + pe;
        double* Gs = a.G + (size_t)s * (s + 1) / 2 * EP + pe;
        const double ps = Ls[(size_t)s * EP];
        const double c = ps > 0.0 ? Gt[(size_t)s * EP] / ps : 0.0;
        for (int r = lane; r < s; r += 32) {
            Gt[(size_t)r * EP] = fma(-c, Ls[(size_t)r * EP], Gt[(size_t)r * EP]);
            Gs[(size_t)r * EP] = fma(-c, Lt[(size_t)r * EP], Gs[(size_t)r * EP]);
        }
        __syncwarp();                                   // every lane has read l_bar_s before it is overwritten
        if (lane == 0) {
            Gs[(size_t)s * EP] = fma(-c, Lt[(size_t)s * EP], Gs[(size_t)s * EP]);
            Gt[(size_t)s * EP] = c;
        }
        __syncwarp();
    }
    // G_ts of step s (s < t: row t; s > t: row s, entry t); 0 at s = t
    auto gts = [&](int s) -> double {
        return s < t ? Gt[(size_t)s * EP] : s > t ? a.G[((size_t)s * (s + 1) / 2 + t) * EP + pe] : 0.0;
    };
    // a_t: lanes stride the columns, 128 at a time; the slots are summed in order
    const double* Kp = a.Kh + pe * np;
    double* Ar = a.A + pe * np;
    for (int j0 = 0; j0 < np; j0 += 128) {
        double acc[4] = {0.0, 0.0, 0.0, 0.0};
        for (int s = 0; s < H; ++s) {
            const double gs = s == t ? -2.0 * db : -gts(s);
            const double* Kr = Kp + (size_t)s * EP * np + j0 + lane;
#pragma unroll
            for (int i = 0; i < 4; ++i) if (j0 + 32 * i + lane < np) acc[i] = fma(gs, Kr[32 * i], acc[i]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) if (j0 + 32 * i + lane < np) Ar[j0 + 32 * i + lane] = acc[i];
    }
    // the direct sum: lane d < D holds dimension d, the kernel distance is fs_cond_kernel's butterfly
    const bool dl = lane < D;
    const double xd = dl ? a.xh[((size_t)t * T + row) * D + lane] : 0.0;
    const double ild = dl ? 1.0 / a.ell[(size_t)e * D + lane] : 0.0;
    const double sf2 = a.sf2[e];
    double ds = 0.0;
    for (int s = 0; s < H; ++s) {
        if (s == t) continue;
        const double xs = dl ? a.xh[((size_t)s * T + row) * D + lane] : 0.0;
        const double q = dl ? (xd - xs) * ild : 0.0;
        const double k = sf2 * exp(-0.5 * fs_bfly(q * q));
        ds = fma(gts(s) * k, xs - xd, ds);
    }
    if (dl) a.dir[pe * D + lane] = ds;
}

// ---- score-function gradient (pilco_particles_rollout_score_grad, DESIGN.md section 16) ----------------------------
// The likelihood-ratio estimator over the forward's transitions, x_t and x_{t+1} held fixed (s_t = sqrt(var_t)):
//   G_t  = sum_{t' > t} step_reward_t' + mult_mu prod_{s <= t} (1 - risk_s) (1 - prod_{s > t} (1 - risk_s)),  t < H-1
//   w_t  = G_t - (S_t - G_t) / (P - 1),  S_t = sum_q G_qt over the restart's particles  (P = 1: w_t = G_t)
//   gmean_t = w_t eps_t / s_t,  gvar_t = w_t (eps_t^2 - 1) / (2 var_t)   (0 where var_t <= 0)
//   x~_bar_t = pilco_gp_predict_vjp at x~_t (the steps do not depend on one another: whole groups of steps per call)
//   z_bar_t = x~_bar_t[Ds:] o maxa e^{-su/2} cos(z_t) (when squashed),  z_bar_{H-1} = 0
// then pg_reduce as after the pathwise sweep.  Box terms enter G, so they enter the gradient.  Joint terms depend on
// the parameters directly through u_t = pi(x_t) even with the states held fixed: pj_grad_kernel adds
// sum_k a_kt d v_k / d u_t to x~_bar_t[Ds:] for every t < H (x~_bar_{H-1} = 0 before it), so z_bar carries the direct term.
struct PsDev : PtPolicy {
    long long T;                                        // R P rows
    const double* eps; const double* traj; const double* step_reward; const double* step_risk;
    const double* var;                                  // [H,T,Ds] the forward's predicted variances
    double* G;                                          // [H-1,T] return-to-go
    double* S;                                          // [R,H] per-(restart, step) sums of G
    double* gmean; double* gvar;                        // [H-1,T,Ds] the VJP's cotangents
    const double* gxt;                                  // [H-1,T,D] the VJP's outputs
    double* zbar;                                       // [T,H,U]
    int direct;                                         // joint terms present: gxt has H steps, z_bar_{H-1} is not 0
};

// grid (ceil(P / 128), R), one thread per particle p of restart r = blockIdx.y: G_t for t = H-2 .. 0 (H > 1).  The
// prefix products are parked in G on the way up; suffix sum and product on the way down, no division.
__global__ void __launch_bounds__(PT_THREADS) ps_togo_kernel(PsDev a) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x;
    if (p >= a.P) return;
    const int H = a.H;
    const size_t row = (size_t)blockIdx.y * a.P + p, T = a.T;
    const double* rw = a.step_reward + row * H;
    const double* rk = a.step_risk + row * H;
    double* G = a.G + row;                              // G_t at G[t T]
    const bool mult = a.n_mult > 0;
    if (mult) {
        double pre = 1.0;
        for (int t = 0; t < H - 1; ++t) { pre *= 1.0 - rk[t]; G[t * T] = pre; }
    }
    double sum = 0.0, suf = 1.0;
    for (int t = H - 2; t >= 0; --t) {
        sum += rw[t + 1];
        double g = sum;
        if (mult) { suf *= 1.0 - rk[t + 1]; g = sum + a.mult_mu * (G[t * T] * (1.0 - suf)); }
        G[t * T] = g;
    }
}

// grid (H-1, R), 256 threads: S_t of restart r = blockIdx.y, step t = blockIdx.x; thread q takes p = q, q + 256, ...
// in order, then pg_block_sum (so a restart's sums do not depend on R)
__global__ void __launch_bounds__(256) ps_base_kernel(PsDev a) {
    PDL_ENTRY();
    __shared__ double red[8], out[1];
    const int t = blockIdx.x, r = blockIdx.y;
    const double* G = a.G + (size_t)t * a.T + (size_t)r * a.P;
    double v[1] = {0.0};
    for (int p = threadIdx.x; p < a.P; p += 256) v[0] += G[p];
    pg_block_sum<1>(v, red, out);
    if (threadIdx.x == 0) a.S[(size_t)r * a.H + t] = out[0];
}

// grid (ceil(P / 128) (H-1), R), one thread per (step t, particle p of restart r = blockIdx.y): the cotangents of
// step t's predict outputs.  eps of particle p is shared by the restarts.
__global__ void __launch_bounds__(PT_THREADS) ps_cot_kernel(PsDev a) {
    PDL_ENTRY();
    const int nb = (a.P + PT_THREADS - 1) / PT_THREADS;
    const int t = blockIdx.x / nb, p = (blockIdx.x % nb) * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= a.P) return;
    const int Ds = a.Ds;
    const size_t row = (size_t)r * a.P + p, tr = (size_t)t * a.T + row;
    const double G = a.G[tr];
    const double w = a.P > 1 ? G - (a.S[(size_t)r * a.H + t] - G) / (a.P - 1) : G;
    const double* ep = a.eps + ((size_t)p * a.H + t) * Ds;
    for (int e = 0; e < Ds; ++e) {
        const double v = a.var[tr * Ds + e], ee = ep[e];
        a.gmean[tr * Ds + e] = v > 0.0 ? w * ee / sqrt(v) : 0.0;
        a.gvar[tr * Ds + e] = v > 0.0 ? w * (ee * ee - 1.0) / (2.0 * v) : 0.0;
    }
}

// grid (ceil(P / 128) H, R), one thread per (step t, particle p of restart r = blockIdx.y): z_bar_t.  z_t is recomputed
// from x_t in pt_step_kernel's order (its policy code, kept as a separate copy for the reason pg_step_kernel gives).
__global__ void __launch_bounds__(PT_THREADS) ps_zbar_kernel(PsDev a) {
    PDL_ENTRY();
    const int nb = (a.P + PT_THREADS - 1) / PT_THREADS;
    const int t = blockIdx.x / nb, p = (blockIdx.x % nb) * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= a.P) return;
    const int Ds = a.Ds, U = a.U, H = a.H;
    const size_t row = (size_t)r * a.P + p;
    double* zb = a.zbar + (row * H + t) * U;
    if (t == H - 1 && !a.direct) {                      // x_H carries no reward
        for (int j = 0; j < U; ++j) zb[j] = 0.0;
        return;
    }
    const double* gx = a.gxt + ((size_t)t * a.T + row) * (Ds + U) + Ds;
    if (!a.squash) {
        for (int j = 0; j < U; ++j) zb[j] = gx[j];
        return;
    }
    const double* xg = a.traj + (row * (H + 1) + t) * Ds;
    double x[MAXD];
#pragma unroll
    for (int d = 0; d < MAXD; ++d) x[d] = d < Ds ? xg[d] : 0.0;
    const double su = a.pol_kind == PILCO_POLICY_RBF ? PT_RBF_VAR : 0.0;
    for (int j = 0; j < U; ++j) {
        double z;
        if (a.pol_kind == PILCO_POLICY_LINEAR) {
            const double* W = a.W + r * a.W_bs;
            z = a.b[r * a.b_bs + j];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < Ds) z = fma(W[j * Ds + d], x[d], z);
        } else {
            const double* ell = a.ell + r * a.ell_bs;
            double il[MAXD];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) il[d] = d < Ds ? 1.0 / ell[j * Ds + d] : 0.0;
            const double sf2 = a.sf2[r * a.sf2_bs + j];
            const double* be = a.beta + r * a.beta_bs + (size_t)j * a.bf;
            const double* C = a.C + r * a.C_bs;
            z = 0.0;
            for (int i = 0; i < a.bf; ++i) {
                const double* c = C + (size_t)i * Ds;
                double d2 = 0.0;
#pragma unroll
                for (int d = 0; d < MAXD; ++d) if (d < Ds) { const double q = (x[d] - c[d]) * il[d]; d2 = fma(q, q, d2); }
                z = fma(sf2 * exp(-0.5 * d2), be[i], z);
            }
        }
        // cos(z) as cospi(z / pi), as pg_step_kernel: no Payne-Hanek slow path and its local-memory table
        zb[j] = gx[j] * (a.maxa[j] * exp(-0.5 * su) * cospi(z * PT_INV_PI));
    }
}

// ---- time-varying linear policy (pilco_particles_scheduled_*, DESIGN.md section 28) ---------------------------------
// Restart r at step t applies W_t = W + r W_bs + t W_ts and b_t = b + r b_bs + t b_ts.  The per-step kernels read the
// policy through their launch's W and b, which the drivers advance by t W_ts and t b_ts; the two kernels below cover
// all H steps in one grid, so they take the step strides themselves.  Linear policies only.
struct PsSched : PsDev {
    long long W_ts, b_ts;
};

// ps_zbar_kernel under a schedule: its grid and its z_bar_t, with z_t from step t's W_t and b_t in pt_step_kernel's
// order.  The linear policy's output variance is 0, so maxa e^{-su/2} is maxa exactly.
__global__ void __launch_bounds__(PT_THREADS) ps_zbar_sched_kernel(PsSched a) {
    PDL_ENTRY();
    const int nb = (a.P + PT_THREADS - 1) / PT_THREADS;
    const int t = blockIdx.x / nb, p = (blockIdx.x % nb) * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= a.P) return;
    const int Ds = a.Ds, U = a.U, H = a.H;
    const size_t row = (size_t)r * a.P + p;
    double* zb = a.zbar + (row * H + t) * U;
    if (t == H - 1 && !a.direct) {                      // x_H carries no reward
        for (int j = 0; j < U; ++j) zb[j] = 0.0;
        return;
    }
    const double* gx = a.gxt + ((size_t)t * a.T + row) * (Ds + U) + Ds;
    if (!a.squash) {
        for (int j = 0; j < U; ++j) zb[j] = gx[j];
        return;
    }
    const double* xg = a.traj + (row * (H + 1) + t) * Ds;
    double x[MAXD];
#pragma unroll
    for (int d = 0; d < MAXD; ++d) x[d] = d < Ds ? xg[d] : 0.0;
    const double* W = a.W + r * a.W_bs + t * a.W_ts;
    const double* b = a.b + r * a.b_bs + t * a.b_ts;
    for (int j = 0; j < U; ++j) {
        double z = b[j];
#pragma unroll
        for (int d = 0; d < MAXD; ++d) if (d < Ds) z = fma(W[j * Ds + d], x[d], z);
        zb[j] = gx[j] * (a.maxa[j] * cospi(z * PT_INV_PI));
    }
}

// The per-step policy-parameter gradient, in place of pg_param_kernel under a schedule: grid (H U + 1, R), 256
// threads.  CTA t U + j of restart r = blockIdx.y forms sum_p z_bar_{p,t,j} [x_{p,t}, 1] over the restart's P
// particles, thread q taking p = q, q + 256, ... in order (so a restart's sums do not depend on R), and writes
// gW [R,H,U,Ds] and gb [R,H,U] over P.  The last CTA is pg_param_kernel's value CTA, the same code.
__global__ void __launch_bounds__(256) pg_sched_kernel(PgRed a) {
    PDL_ENTRY();
    __shared__ double red[(MAXD + 1) * 8], out[MAXD + 1];
    const int Ds = a.Ds, U = a.U, H = a.H, tid = threadIdx.x, r = blockIdx.y;
    const size_t r0 = (size_t)r * a.P;                  // the restart's first row
    const double invP = 1.0 / a.P;
    if ((int)blockIdx.x == H * U) {                     // value = mean return
        double v[1] = {0.0};
        for (int p = tid; p < a.P; p += 256) v[0] += a.ret[r0 + p];
        pg_block_sum<1>(v, red, out);
        if (tid == 0) a.value[r] = out[0] * invP;
        return;
    }
    const int t = blockIdx.x / U, j = blockIdx.x % U;
    const double* traj = a.traj + (r0 * (H + 1) + t) * Ds;          // particle p's x_t at traj[p (H+1) Ds]
    const double* zbar = a.zbar + (r0 * H + t) * U + j;             // its z_bar_{t,j} at zbar[p H U]
    double v[MAXD + 1];
#pragma unroll
    for (int d = 0; d <= MAXD; ++d) v[d] = 0.0;
    for (int p = tid; p < a.P; p += 256) {
        const double* x = traj + (size_t)p * (H + 1) * Ds;
        const double zb = zbar[(size_t)p * H * U];
#pragma unroll
        for (int d = 0; d < MAXD; ++d) if (d < Ds) v[d] = fma(zb, x[d], v[d]);
        v[MAXD] += zb;
    }
    pg_block_sum<MAXD + 1>(v, red, out);
    const size_t o = ((size_t)r * H + t) * U + j;
    if (tid < Ds) a.gW[o * Ds + tid] = out[tid] * invP;
    if (tid == 0) a.gb[o] = out[MAXD] * invP;
}

// ---- host side ------------------------------------------------------------------------------------------------------
// Every entry point is one call of pt_call (or of the query pt_query): pt_validate checks the call once, in one order
// of precedence, and fills a PtOpt; the sampler's layout (pt_ws_layout or fs_ws_layout) places the workspace; the
// forward pt_forward, then pg_reverse (pathwise) or ps_run (score) runs it.

enum PtCall { PT_FORWARD, PT_PATHWISE, PT_SCORE };

// What one validated call runs.  The entry point sets the sampler, the call, batched (and a batched forward's value);
// pt_validate the rest.
struct PtOpt {
    bool consistent;            // one posterior function per particle (DESIGN.md section 14), else step-wise draws
    PtCall call;
    bool batched;               // the policy's batch strides are honoured; otherwise a batched policy is unsupported
    bool resampled;             // the Gaussian refit at every step (DESIGN.md section 26; step-wise sampler only)
    int R;
    bool mapped;                // angles or noise: tm is the angles' map (the identity without angles)
    TrigMap tm;
    bool noisy;                 // measurement noise (DESIGN.md section 23)
    PnNoise nz;
    bool explore, bonus;        // exploration (section 24): the moments; bonus (b != 0): its share and its value
    double b;
    double* step_var;
    pilco_particles_resample rs;
    bool sched;                 // an active schedule (DESIGN.md section 28): step t's linear policy at t sch strides
    pilco_policy_schedule sch;
    bool mlp;                   // an MLP call (DESIGN.md section 29): the policy is net, pol.kind must be PILCO_POLICY_MLP
    PmNet net;
    bool features;              // function samples from random-feature draws (DESIGN.md section 30): fd's, not eps
    pilco_feature_draws fd;
    double* value;              // a batched forward (call PT_FORWARD with batched, DESIGN.md section 31): the mean
                                // return per restart [R], set by the entry point
};

// Offsets in doubles into a particle workspace, for both layouts (a slot a call does not have stays 0); the predict
// (pws) and VJP (vws) workspaces are one slot when one call needs both.  total in bytes; 0 for unsupported sizes and
// on size_t overflow.
struct PtWs {
    size_t xt, mean, var;                               // forward: x~ [H or 1,T,D], step closure mean [T,Ds], var
    size_t mu, s2, W, Kh, L;                            // consistent forward: predict outputs, W_t, K* history, factor
    size_t gx, gvar, gxt, zbar, s1, s2r, gbeta, gy;     // reverse sweep and the policy-parameter reduction
    size_t G, dir;                                      // consistent: reverse of the conditioning
    size_t phi;                                         // angles, gradients: phi(x_t) [T,H+1,Dh]
    size_t phiz, phibz;                                 // noise, gradients: phi(z_t) [T,H+1,Dh]; phi_bar_z [T,Dh]
    size_t sd, tab;                                     // exploration: sigma_t [R,H]; the bonus table [R,H,K,2]
    size_t togo, gsum, mw, vw, gxh;                     // score: G [H-1,T]; the sums [R,H]; m_bar, v_bar [H-1,T,E];
                                                        // the x~_bar history [H-1 or H,T,D]
    size_t xp, rmu, rL, rsc;                            // resampled: x' [H,T,Ds], mu^ [H,R,Ds], L^ [H,R,Ds,Ds]; the
                                                        // reverse scratch [R,Ds+Ds Ds]
    size_t min0, min1, min2, md1, md2, mdo, mpart;      // MLP, gradients: the layer inputs and cotangents [., R Pp];
                                                        // the chunk partials [R nc, n_theta]
    size_t fz;                                          // features: the zero eps [P,H,Ds] the step kernels read
    size_t pws, pws_bytes, vws, vws_bytes, total;
};

// slots of dims[0] x dims[1] x ... doubles, each rounded up to an even count (16 bytes); ok = false on size_t overflow
struct PtTake {
    size_t o = 0;
    bool ok = true;
    size_t operator()(std::initializer_list<size_t> dims) {
        size_t len = 1;
        for (size_t d : dims) ok = ok && !__builtin_mul_overflow(len, d, &len);
        const size_t at = o;
        ok = ok && !__builtin_add_overflow(len, len & 1, &len) && !__builtin_add_overflow(o, len, &o);
        return at;
    }
    size_t bytes() { size_t b = 0; return ok && !__builtin_mul_overflow(o, sizeof(double), &b) ? b : 0; }
};

static bool pt_rbf(const pilco_particles* pr) { return pr->pol.kind == PILCO_POLICY_RBF; }
static bool pt_has_joint(const pilco_particles* pr) {
    for (int k = 0; k < pr->n_rewards && k < 8; ++k) if (reward_on_joint(pr->rewards[k].kind)) return true;
    return false;
}

// steps per pilco_gp_predict_vjp call of the score gradient: whole steps of T rows, at most PT_MAX_P rows (T <= PT_MAX_P)
static int ps_group(long long T, int H) {
    const long long k = PT_MAX_P / T;
    return H - 1 < k ? H - 1 : (int)k;
}

// The MLP reduction's chunks of a restart's P rows: Kc rows each (a multiple of 16, the gemm's k tile), nc <= PM_CHUNKS
// of them, Pp = nc Kc rows with the padding
struct PmChunks {
    int Kc, nc;
    long long Pp;
};
static PmChunks pm_chunks(int P) {
    PmChunks c;
    const int per = (P + PM_CHUNKS - 1) / PM_CHUNKS;
    c.Kc = (per + 15) / 16 * 16;
    c.nc = (P + c.Kc - 1) / c.Kc;
    c.Pp = (long long)c.nc * c.Kc;
    return c;
}

// the MLP gradient's slots, after every other slot: [x; 1], [h_1; 1], [h_2; 1], d_1, d_2, d_out, each [width, R Pp],
// contiguous (one memset clears them), then the chunk partials [R nc, n_theta]
static void pm_ws_slots(PtWs& L, PtTake& take, const pilco_particles* pr, const PtOpt& o) {
    const PmNet& m = o.net;
    const PmChunks c = pm_chunks(pr->P);
    const size_t RPp = (size_t)o.R * c.Pp, Dh = pr->pol.Ds, U = pr->pol.U, w1 = m.w1, w2 = m.w2;
    L.min0 = take({Dh + 1, RPp}); L.min1 = take({w1 + 1, RPp}); L.min2 = take({m.L == 2 ? w2 + 1 : 0, RPp});
    L.md1 = take({w1, RPp}); L.md2 = take({w2, RPp}); L.mdo = take({U, RPp});
    L.mpart = take({(size_t)o.R * c.nc, (size_t)m.n_theta});
}

// The step-wise sampler's workspace at T = R P rows (restart-major, row r P + p; nothing of size [., n] is kept).
// State-width slots are in dyn.E, the RBF sums in the policy's width pol.Ds (the same without angles).
//   forward-only: x~ [T,D], the step closure's mean and var [T,Ds], one predict workspace at T
//   pathwise: x~ and var of EVERY step [H,T,D] and [H,T,Ds] (the reverse sweep needs them), mean [T,Ds], x_bar and
//     var_bar [T,Ds], the VJP output [T,D], z_bar [T,H,U], the RBF sums [R,U,bf,Dh] x 2 and [R,U,bf] x 2, and one
//     predict / VJP workspace at T (never in use at the same time)
//   score (DESIGN.md section 16): as pathwise, but G [H-1,T], the sums [R,H], m_bar and v_bar [H-1,T,Ds] and the VJP
//     output [H-1,T,D] (joint terms: [H,T,D]) in place of x_bar .. the VJP output, and the VJP workspace for the
//     largest VJP group; 0 also where the per-(step, particle) grids would pass 2^31 - 1 CTAs
// then, gradients only: the phi history [T,H+1,Dh] (angles or noise); the phi(z) history [T,H+1,Dh] and (pathwise)
// phi_bar_z [T,Dh] (noise); sigma_t [R,H] and the bonus table [R,H,K,2] (exploration, K = n_rewards).
// Resampled (DESIGN.md section 26), after every other slot: the x' history [H,T,Ds], mu^ [H,R,Ds], L^ [H,R,Ds,Ds] and,
// gradients only, the reverse scratch [R,Ds+Ds Ds].
static PtWs pt_ws_layout(const pilco_particles* pr, const PtOpt& o) {
    const bool grad = o.call != PT_FORWARD, score = o.call == PT_SCORE;
    const size_t R = o.R, T = R * pr->P, H = pr->H, Hm = H > 0 ? H - 1 : 0, Hx = grad ? H : 1;
    const size_t Ds = pr->dyn.E, Dh = pr->pol.Ds, U = pr->pol.U, D = pr->dyn.D, bf = pt_rbf(pr) ? pr->pol.rbf.n : 0;
    PtWs L = {}; PtTake take;
    L.xt = take({Hx, T, D}); L.mean = take({T, Ds}); L.var = take({Hx, T, Ds});
    if (score) {
        L.togo = take({Hm, T}); L.gsum = take({R, H});
        L.mw = take({Hm, T, Ds}); L.vw = take({Hm, T, Ds});
        L.gxh = take({pt_has_joint(pr) ? H : Hm, T, D});    // joint terms: step H-1 too, for their direct term
    } else if (grad) {
        L.gx = take({T, Ds}); L.gvar = take({T, Ds}); L.gxt = take({T, D});
    }
    if (grad) {
        L.zbar = take({T, H, o.mlp ? 0 : U});
        L.s1 = take({R, U, bf, Dh}); L.s2r = take({R, U, bf, Dh});
        L.gbeta = take({R, U, bf}); L.gy = take({R, U, bf});
    }
    const int grp = score ? ps_group((long long)T, (int)H) : 1;
    const size_t pb = pilco_gp_predict_workspace_bytes(pr->dyn.n, pr->dyn.D, (int)Ds, (int)T, 0);
    const size_t vb = grad ? pilco_gp_predict_vjp_workspace_bytes(pr->dyn.n, pr->dyn.D, pr->dyn.E,
                                                                  (int)T * (grp > 1 ? grp : 1)) : pb;
    L.pws_bytes = L.vws_bytes = (pb && vb) ? (pb > vb ? pb : vb) : 0;
    L.pws = L.vws = take({L.pws_bytes / sizeof(double)});
    if (grad && o.mapped) L.phi = take({T, H + 1, Dh});
    if (grad && o.noisy) { L.phiz = take({T, H + 1, Dh}); if (!score) L.phibz = take({T, Dh}); }
    if (o.explore) { L.sd = take({R, H}); L.tab = take({R, H, (size_t)pr->n_rewards, 2}); }
    if (o.resampled) {
        L.xp = take({H, T, Ds}); L.rmu = take({H, R, Ds}); L.rL = take({H, R, Ds, Ds});
        if (grad) L.rsc = take({R, Ds + Ds * Ds});
    }
    if (grad && o.mlp) pm_ws_slots(L, take, pr, o);
    const size_t nb = (pr->P + PT_THREADS - 1) / PT_THREADS;
    L.total = L.pws_bytes && (!score || nb * H <= 0x7fffffff) ? take.bytes() : 0;
    return L;
}

// The consistent sampler's workspace at T = R P rows (DESIGN.md sections 14, 15, 25):
//   forward: x~ of every step [H,T,D], the predict outputs mu and var and the step closure's mean and var [T,Ds], W_t
//     [E,T,np], the K* history [H,E,T,np], the packed factor rows [H(H+1)/2,E,T], one predict workspace at T
//   gradients: then the var' history [H,T,Ds], the packed cotangent rows [H(H+1)/2,E,T], the direct sums [E,T,D],
//     x_bar and var_bar [T,Ds], the VJP output [T,D], z_bar [T,H,U], the RBF sums [R,U,bf,Ds] x 2 and [R,U,bf] x 2,
//     and one VJP workspace at T (the W slot holds a_t in the reverse sweep); then the phi history (angles or noise),
//     the phi(z) history and phi_bar_z (noise), sigma_t and the bonus table (exploration), as pt_ws_layout
//   score: then G [H-1,T], the sums [R,H], m_bar and v_bar [H-1,T,E] and the x~_bar history [H,T,D]; 0 also where
//     the per-(step, particle) grids would pass 2^31 - 1 CTAs
static PtWs fs_ws_layout(const pilco_particles* pr, const PtOpt& o) {
    const bool grad = o.call != PT_FORWARD, score = o.call == PT_SCORE;
    const size_t R = o.R, T = R * pr->P, H = pr->H, Hm = H > 0 ? H - 1 : 0, np = (size_t)pad64(pr->dyn.n);
    const size_t Ds = pr->dyn.E, Dh = pr->pol.Ds, U = pr->pol.U, D = pr->dyn.D, bf = pt_rbf(pr) ? pr->pol.rbf.n : 0;
    PtWs L = {}; PtTake take;                           // pt_batch_ok: R P <= PT_MAX_P
    L.xt = take({H, T, D}); L.mu = take({T, Ds}); L.s2 = take({T, Ds}); L.mean = take({T, Ds}); L.var = take({T, Ds});
    L.W = take({T, Ds, np}); L.Kh = take({H, T, Ds, np}); L.L = take({H * (H + 1) / 2, T, Ds});
    L.pws_bytes = pilco_gp_predict_workspace_bytes(pr->dyn.n, pr->dyn.D, (int)Ds, (int)T, 0);
    L.pws = take({L.pws_bytes / sizeof(double)});
    bool grids = true;
    if (grad) {
        // the var' history supersedes the forward's var slot, whose bytes stay: the sizes reported for these calls
        // include them
        L.var = take({H, T, Ds}); L.G = take({H * (H + 1) / 2, T, Ds}); L.dir = take({T, Ds, D});
        L.gx = take({T, Ds}); L.gvar = take({T, Ds}); L.gxt = take({T, D}); L.zbar = take({T, H, o.mlp ? 0 : U});
        L.s1 = take({R, U, bf, Dh}); L.s2r = take({R, U, bf, Dh});
        L.gbeta = take({R, U, bf}); L.gy = take({R, U, bf});
        L.vws_bytes = pilco_gp_predict_vjp_workspace_bytes(pr->dyn.n, pr->dyn.D, pr->dyn.E, (int)T);
        L.vws = take({L.vws_bytes / sizeof(double)});
        if (o.mapped) L.phi = take({T, H + 1, Dh});
        if (o.noisy) { L.phiz = take({T, H + 1, Dh}); L.phibz = take({T, Dh}); }
        if (o.explore) { L.sd = take({R, H}); L.tab = take({R, H, (size_t)pr->n_rewards, 2}); }
        if (score) {
            const size_t nb = (pr->P + PT_THREADS - 1) / PT_THREADS;
            L.togo = take({Hm, T}); L.gsum = take({R, H});
            L.mw = take({Hm, T, Ds}); L.vw = take({Hm, T, Ds}); L.gxh = take({H, T, D});
            grids = nb * H <= 0x7fffffff;
        }
        if (o.mlp) pm_ws_slots(L, take, pr, o);
    }
    L.total = L.pws_bytes && (!grad || L.vws_bytes) && grids ? take.bytes() : 0;
    return L;
}

// The feature sampler's workspace at T = R P rows (DESIGN.md section 30): pt_ws_layout's forward and pathwise slots
// without the predict and VJP workspaces, then the zero eps [P,H,Ds] with which the unchanged step kernels close each
// step (x + f + sqrt(0) 0 = x + f exactly).
static PtWs pf_ws_layout(const pilco_particles* pr, const PtOpt& o) {
    const bool grad = o.call != PT_FORWARD;
    const size_t R = o.R, T = R * pr->P, H = pr->H, Hx = grad ? H : 1;
    const size_t Ds = pr->dyn.E, Dh = pr->pol.Ds, U = pr->pol.U, D = pr->dyn.D, bf = pt_rbf(pr) ? pr->pol.rbf.n : 0;
    PtWs L = {}; PtTake take;
    L.xt = take({Hx, T, D}); L.mean = take({T, Ds}); L.var = take({Hx, T, Ds});
    if (grad) {
        L.gx = take({T, Ds}); L.gvar = take({T, Ds}); L.gxt = take({T, D}); L.zbar = take({T, H, o.mlp ? 0 : U});
        L.s1 = take({R, U, bf, Dh}); L.s2r = take({R, U, bf, Dh});
        L.gbeta = take({R, U, bf}); L.gy = take({R, U, bf});
        if (o.mapped) L.phi = take({T, H + 1, Dh});
        if (o.noisy) { L.phiz = take({T, H + 1, Dh}); L.phibz = take({T, Dh}); }
        if (o.explore) { L.sd = take({R, H}); L.tab = take({R, H, (size_t)pr->n_rewards, 2}); }
    }
    L.fz = take({(size_t)pr->P, H, Ds});
    if (grad && o.mlp) pm_ws_slots(L, take, pr, o);
    L.total = take.bytes();
    return L;
}

static PtWs pt_layout(const pilco_particles* pr, const PtOpt& o) {
    return o.features ? pf_ws_layout(pr, o) : o.consistent ? fs_ws_layout(pr, o) : pt_ws_layout(pr, o);
}

static bool pt_sizes_ok(const pilco_particles* pr) {
    return pr->P >= 1 && pr->P <= PT_MAX_P && pr->H >= 0 && pr->dyn.n >= 1 && pr->dyn.D >= 1 && pr->dyn.D <= MAXD &&
           pr->pol.Ds >= 1 && pr->pol.U >= 1 && pr->pol.Ds <= MAXE;
}

// R restarts of P particles: one CTA row per restart (gridDim.y) and R P predict points
static bool pt_batch_ok(int P, int R) {
    return R >= 1 && R <= 65535 && (long long)R * P <= PT_MAX_P;
}

// the reward terms: their count, then each term's W, kind, channel and t (no_additive_box: an ADD-channel box term is
// unsupported, section 21's rule for the reward's sample moments)
static int pt_check_rewards(const pilco_particles* pr, bool no_additive_box) {
    if (pr->n_rewards < 1 || pr->n_rewards > 8) return PILCO_ERR_DIM;
    for (int k = 0; k < pr->n_rewards; ++k) {
        const pilco_reward_term& rt = pr->rewards[k];
        if (!rt.W) return PILCO_ERR_NULL;
        if (!reward_kind_known(rt.kind)) return PILCO_ERR_UNSUPPORTED;
        if (rt.channel != PILCO_CHANNEL_ADD && rt.channel != PILCO_CHANNEL_MULT) return PILCO_ERR_UNSUPPORTED;
        if (reward_needs_t(rt.kind) && !rt.t) return PILCO_ERR_NULL;
        if (no_additive_box && rt.channel == PILCO_CHANNEL_ADD && rt.kind == PILCO_REWARD_BOX)
            return PILCO_ERR_UNSUPPORTED;
    }
    return PILCO_OK;
}

// an MLP's sizes: L in {1, 2}, each hidden width in 1 .. PM_MAXW
static bool pm_sizes_ok(const pilco_mlp* m) {
    if (m->L < 1 || m->L > 2) return false;
    for (int l = 0; l < m->L; ++l) if (m->width[l] < 1 || m->width[l] > PM_MAXW) return false;
    return true;
}

// the MLP's device description (sizes checked): theta's length and block offsets
static PmNet pm_net(const pilco_particles* pr, const pilco_mlp* m) {
    PmNet n;
    const int Ds = pr->pol.Ds, U = pr->pol.U;
    n.L = m->L; n.w1 = m->width[0]; n.w2 = m->L == 2 ? m->width[1] : 0;
    n.off2 = n.w1 * (Ds + 1);
    n.offo = n.off2 + (m->L == 2 ? n.w2 * (n.w1 + 1) : 0);
    n.n_theta = n.offo + U * ((m->L == 2 ? n.w2 : n.w1) + 1);
    n.theta = m->theta; n.theta_bs = m->theta_bs;
    return n;
}

// everything but the workspace (the gradients bring their own).  batched: the policy's batch strides are honoured
// (the batch_grad and consistent_grad entry points); otherwise a batched policy is unsupported.  A: the number of
// angular state dimensions (the policy takes dyn.E + A inputs).  mlp_call: the MLP entry points, whose policy checks
// are the MLP's (pol.kind PILCO_POLICY_MLP, mlp and theta not NULL, its sizes, theta_bs as a batch stride).  need_eps
// = false (the feature sampler): pr->eps is not read and may be NULL.
static int pt_check_desc(const pilco_particles* pr, bool batched = false, int A = 0, bool mlp_call = false,
                         const pilco_mlp* mlp = nullptr, bool need_eps = true) {
    if (!pr) return PILCO_ERR_NULL;
    if (pr->P < 1 || pr->P > PT_MAX_P || pr->H < 0) return PILCO_ERR_DIM;
    const pilco_gp_model& g = pr->dyn;
    if (!g.X || !g.ell || !g.sf2 || !g.beta) return PILCO_ERR_NULL;
    if (g.mode != 0 || !g.iK || g.X_bs || g.ell_bs || g.sf2_bs || g.beta_bs) return PILCO_ERR_UNSUPPORTED;
    if (g.n < 1 || g.D < 1 || g.D > MAXD || g.E < 1 || g.E > MAXE || g.ldk < pad64(g.n)) return PILCO_ERR_DIM;
    const pilco_policy& pol = pr->pol;
    const int Ds = pol.Ds, U = pol.U;
    if (Ds < 1 || U < 1 || Ds + U != g.D || g.E + A != Ds) return PILCO_ERR_DIM;
    auto strides = [batched](std::initializer_list<long long> bs) {
        for (long long b : bs) {
            if (b && !batched) return PILCO_ERR_UNSUPPORTED;
            if (b < 0) return PILCO_ERR_DIM;
        }
        return PILCO_OK;
    };
    if (mlp_call) {
        if (pol.kind != PILCO_POLICY_MLP) return PILCO_ERR_UNSUPPORTED;
        if (!mlp || !mlp->theta) return PILCO_ERR_NULL;
        if (!pm_sizes_ok(mlp) || mlp->theta_bs < 0) return PILCO_ERR_DIM;
        if (const int rc = strides({mlp->theta_bs})) return rc;
    } else if (pol.kind == PILCO_POLICY_LINEAR) {
        if (!pol.W || !pol.b) return PILCO_ERR_NULL;
        if (const int rc = strides({pol.W_bs, pol.b_bs})) return rc;
    } else if (pol.kind == PILCO_POLICY_RBF) {
        const pilco_gp_model& r = pol.rbf;
        if (!r.X || !r.ell || !r.sf2 || !r.beta) return PILCO_ERR_NULL;
        if (r.mode != 1) return PILCO_ERR_UNSUPPORTED;
        if (const int rc = strides({r.X_bs, r.ell_bs, r.sf2_bs, r.beta_bs})) return rc;
        if (r.n < 1 || r.D != Ds || r.E != U) return PILCO_ERR_DIM;
    } else return PILCO_ERR_UNSUPPORTED;
    if (pol.squash && !pol.max_action) return PILCO_ERR_NULL;
    if (const int rc = pt_check_rewards(pr, false)) return rc;
    if (!pr->x0 || (need_eps && !pr->eps) || !pr->traj || !pr->act || !pr->step_reward || !pr->step_risk || !pr->ret)
        return PILCO_ERR_NULL;
    if (((uintptr_t)g.iK & 15) || (g.ldk & 1)) return PILCO_ERR_ALIGN;                  // predict's TMA rows
    return PILCO_OK;
}

// a workspace against its layout's total (0: unsupported sizes)
static int pt_check_ws(const void* ws, size_t ws_bytes, size_t total) {
    if (!ws) return PILCO_ERR_NULL;
    if ((uintptr_t)ws & 15) return PILCO_ERR_ALIGN;
    if (total == 0) return PILCO_ERR_DIM;
    if (ws_bytes < total) return PILCO_ERR_WORKSPACE;
    return PILCO_OK;
}

// the gradient's output pointers, after pt_check_desc (mlp: the MLP's gtheta in place of the policy's fields)
static int pg_check(const pilco_particles* pr, const pilco_particles_grad* g, const pilco_mlp* mlp = nullptr) {
    if (!g || !g->value || !g->ws) return PILCO_ERR_NULL;
    if (mlp) return mlp->gtheta ? PILCO_OK : PILCO_ERR_NULL;
    if (pt_rbf(pr) ? (!g->gXc || !g->gYc || !g->gell || !g->pol_L) : (!g->gW || !g->gb)) return PILCO_ERR_NULL;
    return PILCO_OK;
}

// joint = false: the state terms, for the per-particle state kernels; true: the joint state-action terms, for
// pt_joint_kernel / pj_grad_kernel.  n_mult counts the MULT terms of both.
static PtPolicy pt_policy(const pilco_particles* pr, bool joint = false) {
    const pilco_policy& pol = pr->pol;
    const bool rbf = pol.kind == PILCO_POLICY_RBF;
    PtPolicy a;
    a.P = pr->P; a.H = pr->H; a.Ds = pol.Ds; a.U = pol.U;
    a.pol_kind = pol.kind; a.squash = pol.squash; a.maxa = pol.max_action;
    a.W = pol.W; a.b = pol.b;
    a.C = pol.rbf.X; a.ell = pol.rbf.ell; a.sf2 = pol.rbf.sf2; a.beta = pol.rbf.beta; a.bf = rbf ? pol.rbf.n : 0;
    a.W_bs = rbf ? 0 : pol.W_bs; a.b_bs = rbf ? 0 : pol.b_bs;
    a.C_bs = rbf ? pol.rbf.X_bs : 0; a.ell_bs = rbf ? pol.rbf.ell_bs : 0;
    a.sf2_bs = rbf ? pol.rbf.sf2_bs : 0; a.beta_bs = rbf ? pol.rbf.beta_bs : 0;
    a.n_rewards = 0; a.n_mult = 0;
    for (int k = 0; k < 8; ++k) a.rewards[k] = pilco_reward_term();
    for (int k = 0; k < pr->n_rewards; ++k) {
        if (reward_on_joint(pr->rewards[k].kind) == joint) a.rewards[a.n_rewards++] = pr->rewards[k];
        a.n_mult += pr->rewards[k].channel == PILCO_CHANNEL_MULT;
    }
    a.mult_mu = pr->mult_mu;
    return a;
}

static PjDev pj_dev(const pilco_particles* pr, int R) {
    PjDev j;
    static_cast<PtPolicy&>(j) = pt_policy(pr, true);
    j.T = (long long)R * pr->P; j.t = 0; j.xh = nullptr;
    j.step_reward = pr->step_reward; j.step_risk = pr->step_risk;
    j.gxt = nullptr; j.gstep = 0; j.first = 0;
    return j;
}

int fs_predict_prepare();
int fs_predict_launch(cudaStream_t st, const pilco_gp_model* gp, int T, const double* Xs, double* mean, double* var,
                      double* W, double* Ks, void* ws);
int fs_vjp_prepare();
int fs_vjp_launch(cudaStream_t st, const pilco_gp_model* gp, int T, const double* Xs, const double* gmean,
                  const double* A, const double* dir, double* gXs, void* ws);

// The forward of every entry point, R restarts (validated; T = R P rows):
//   pt_step<0>, predict<0>, [fs_cond<0>,] pt_step<1>, ..., pt_step<H>
// consistent: the predict is fs_predict_kernel and fs_cond_kernel leaves the step closure (mean, var) that
// pt_step_kernel reads unchanged.  history: var of every step is kept (the reverse sweep needs it); x~ of every step is
// kept when either needs it.  tm (angles, DESIGN.md section 20): pa_step_kernel in place of pt_step_kernel, which with
// history also keeps phi(x_t) in L.phi.  nz (noise, DESIGN.md section 23; tm then given, the identity without angles):
// pn_step_kernel in place of pa_step_kernel, which with history also keeps phi(z_t) in L.phiz.  The state width is
// dyn.E throughout (pol.Ds without angles).  sch (an active schedule, DESIGN.md section 28): every step kernel reads
// the linear policy through a.W and a.b, which step t's launch advances by t W_ts and t b_ts.  net (an MLP, DESIGN.md
// section 29; no angles, noise or schedule): pm_step_kernel / pm_refit_kernel in place of pt_step / pr_step.  pf
// (feature draws, DESIGN.md section 30; not consistent, no refit or schedule): pf_eval_kernel in place of the predict,
// and the step kernels read the zero eps in L.fz.
static int pt_forward(const pilco_particles* pr, int R, double* ws, const PtWs& L, bool consistent, bool history,
                      cudaStream_t st, const TrigMap* tm = nullptr, const PnNoise* nz = nullptr,
                      const pilco_particles_resample* rs = nullptr, const pilco_policy_schedule* sch = nullptr,
                      const PmNet* net = nullptr, const PfDev* pf = nullptr) {
    const int P = pr->P, H = pr->H, Ds = pr->dyn.E, D = pr->dyn.D, T = R * P, np = pad64(pr->dyn.n);
    const size_t TD = (size_t)T * D, TDs = (size_t)T * Ds, slot = TDs * np;
    const size_t xstep = consistent || history ? TD : 0, vstep = history ? TDs : 0;
    const dim3 grid((P + PT_THREADS - 1) / PT_THREADS, R), cgrid((P + FS_WARPS - 1) / FS_WARPS, Ds, R);
    PtDev a;
    static_cast<PtPolicy&>(a) = pt_policy(pr);
    a.x0 = pr->x0; a.eps = pf ? ws + L.fz : pr->eps;
    if (pf && H > 0) cudaMemsetAsync(ws + L.fz, 0, (size_t)P * H * Ds * sizeof(double), st);
    a.traj = pr->traj; a.act = pr->act; a.step_reward = pr->step_reward; a.step_risk = pr->step_risk; a.ret = pr->ret;
    a.mean = ws + L.mean;
    PaStep pa;
    if (tm) { pa.E = Ds; pa.tm = *tm; pa.phi = history ? ws + L.phi : nullptr; }
    PnStep pn;
    if (nz) { pn.nz = *nz; pn.phiz = history ? ws + L.phiz : nullptr; }
    FsCond c;
    c.P = P; c.T = T; c.H = H; c.D = D; c.Ds = Ds; c.n = pr->dyn.n; c.np = np; c.t = 0;
    c.ell = pr->dyn.ell; c.sf2 = pr->dyn.sf2;
    c.xh = ws + L.xt; c.mu = ws + L.mu; c.s2 = ws + L.s2; c.W = ws + L.W; c.Kh = ws + L.Kh;
    c.eps = pr->eps; c.L = ws + L.L; c.mean = ws + L.mean;
    const bool joint = pt_has_joint(pr);
    PjDev j = pj_dev(pr, R);
    PrFwd f;
    if (rs) {
        f.P = P; f.H = H; f.Ds = Ds; f.x0 = pr->x0; f.xi = rs->xi;
        f.xp = ws + L.xp; f.mu = ws + L.rmu; f.L = ws + L.rL; f.step_mean = rs->step_mean; f.step_cov = rs->step_cov;
    }
    for (int t = 0; t <= H; ++t) {
        a.t = t;
        if (sch) { a.W = pr->pol.W + (t < H ? t : 0) * sch->W_ts; a.b = pr->pol.b + (t < H ? t : 0) * sch->b_ts; }
        a.xt = ws + L.xt + (size_t)(t < H ? t : 0) * xstep;
        a.var = ws + L.var + (size_t)(t > 0 ? t - 1 : 0) * vstep;
        if (rs && t > 0) {
            if (const int rc = pr_step_launch(st, grid, a, f, net)) return rc;
        } else if (nz) {
            static_cast<PtDev&>(pa) = a;
            static_cast<PaStep&>(pn) = pa;
            if (const int rc = pn_step_launch(st, grid, pn)) return rc;
        } else if (tm) {
            static_cast<PtDev&>(pa) = a;
            if (const int rc = pa_step_launch(st, grid, pa)) return rc;
        } else {
            if (net) {
                if (const int rc = pm_step_launch(st, grid, a, *net)) return rc;
            } else {
                launch_hi(pt_step_kernel, grid, dim3(PT_THREADS), 0, st, a);
                CUDA_LAUNCH_CHECK();
            }
            if (rs)                                     // t = 0: the moments of x0
                if (const int rc = pr_step_launch(st, grid, a, f)) return rc;
        }
        if (t == H) break;
        if (joint) {
            j.t = t; j.xh = a.xt;
            launch_hi(pt_joint_kernel, grid, dim3(PT_THREADS), 0, st, j);
            CUDA_LAUNCH_CHECK();
        }
        double* var = ws + L.var + (size_t)t * vstep;
        if (consistent) {
            const int rc = fs_predict_launch(st, &pr->dyn, T, a.xt, ws + L.mu, ws + L.s2, ws + L.W, ws + L.Kh + t * slot,
                                             ws + L.pws);
            if (rc) return rc;
            c.t = t; c.var = var;
            launch_hi(fs_cond_kernel, cgrid, dim3(FS_WARPS * 32), 0, st, c);
            CUDA_LAUNCH_CHECK();
        } else if (pf) {
            PfDev q = *pf;
            q.xh = a.xt; q.mean = ws + L.mean; q.var = var;
            if (const int rc = pf_eval_launch(st, q)) return rc;
        } else {
            const int rc = pilco_gp_predict(&pr->dyn, 0, Ds, T, a.xt, ws + L.mean, var, 0, ws + L.pws, L.pws_bytes, st);
            if (rc) return rc;
        }
    }
    return PILCO_OK;
}

int chol_solve_vec_launch(cudaStream_t st, int batch, int n, const double* L, int ld, long long ms, int E,
                          const double* Y, long long Y_bs, long long y_es, int yinc, double* x, long long xs);
int rbf_factor_bwd_launch(cudaStream_t st, int R, int bf, int Ds, int U, const double* X, long long X_bs,
                          const double* ell, long long ell_bs, const double* sf2, long long sf2_bs,
                          const double* beta, long long beta_bs, const double* gy,
                          double* gX, double* gY, double* gell);

// value and the policy-parameter gradient over all P H points of each restart, fixed order, from z_bar [R P,H,U] and
// the policy inputs pin [R P,H+1,Ds] (pr->traj, or with angles the phi history); sched: per step (pg_sched_kernel)
static int pg_reduce(const pilco_particles* pr, int R, const pilco_particles_grad* g, double* ws, const PtWs& L,
                     cudaStream_t st, const double* pin, bool sched = false) {
    PgRed r;
    static_cast<PtPolicy&>(r) = pt_policy(pr);
    const bool rbf = r.pol_kind == PILCO_POLICY_RBF;
    const int Ds = r.Ds, U = r.U, bf = r.bf;
    r.traj = pin; r.zbar = ws + L.zbar; r.ret = pr->ret;
    r.gW = g->gW; r.gb = g->gb;
    r.s1 = ws + L.s1; r.s2 = ws + L.s2r; r.gbeta = ws + L.gbeta;
    r.gXc = g->gXc; r.gell = g->gell;
    r.value = g->value;
    if (sched) {                                        // linear (pt_validate)
        launch_hi(pg_sched_kernel, dim3(r.H * U + 1, R), dim3(256), 0, st, r);
        CUDA_LAUNCH_CHECK();
        return PILCO_OK;
    }
    launch_hi(pg_param_kernel, dim3((rbf ? U * bf : U) + 1, R), dim3(256), 0, st, r);
    CUDA_LAUNCH_CHECK();
    if (rbf) {                                          // through beta = (K + sn2 I)^-1 Yc, as pilco_rollout_backward
        const int ldw = pad64(bf);
        launch_hi(pg_rbf_finish_kernel, dim3(R), dim3(128), 0, st, r);
        CUDA_LAUNCH_CHECK();
        if (const int rcs = chol_solve_vec_launch(st, R * U, bf, g->pol_L, ldw, (long long)ldw * ldw, U,
                                                  r.gbeta, (long long)U * bf, bf, 1, ws + L.gy, bf)) return rcs;
        const int rc = rbf_factor_bwd_launch(st, R, bf, Ds, U, r.C, r.C_bs, r.ell, r.ell_bs, r.sf2, r.sf2_bs,
                                             r.beta, r.beta_bs, ws + L.gy, g->gXc, g->gYc, g->gell);
        if (rc) return rc;
    }
    return PILCO_OK;
}

// The reverse sweep after pt_forward(history) and the reduction (DESIGN.md sections 12, 15):
//   pg_step<H-1>, [VJP<t>, pg_step<t>] for t = H-2 .. 0, then pg_reduce's launches
// The step's VJP is pilco_gp_predict_vjp, or (consistent) fs_cond_bwd_kernel followed by fs_predict_vjp_kernel.
// tm (angles): pa_reverse_launch's two kernels in place of pg_step, and the policy reduction over the phi history.
// nz (noise): pn_reverse_launch's two kernels, and the policy reduction over the phi(z) history.
// bonus (exploration, b != 0): px_bonus_kernel after each step's VJP (and pj_grad) adds the bonus's share to x_bar_{t+1}
// and x~_bar_t, which the step kernel then carries into x_bar_t; the sweep starts as with joint terms (x_bar_H = 0 and
// x~_bar_{H-1} = 0 passed to the step kernel, which ignores x_bar when x~_bar is NULL).
// rs (resampled): after the step kernel of each t = H-1 .. 1, pr_reverse_launch turns x_bar_t (the cotangent of the
// refitted particles) into that of x'_t and rewrites var_bar_{t-1}.
// sch (an active schedule): the step kernels of step t read W_t and b_t as pt_forward's, and the reduction is per step.
// net (an MLP): pm_reverse_kernel in place of pg_step, then (where x~_bar_t exists) one gemm per layer adds step t's
// d_l' [a_{l-1}; 1] to each chunk's partial, steps in order t = H-1 .. 0; pm_finish_kernel sums the chunks over P into
// gtheta and writes value.
// pf (feature draws): pf_vjp_kernel is the step's VJP (var = 0, so var_bar has no share), and the step kernels read
// the forward's zero eps.
static int pg_reverse(const pilco_particles* pr, int R, const pilco_particles_grad* g, const PtWs& L, bool consistent,
                      cudaStream_t st, const TrigMap* tm = nullptr, const PnNoise* nz = nullptr, bool bonus = false,
                      const pilco_particles_resample* rs = nullptr, const pilco_policy_schedule* sch = nullptr,
                      const PmNet* net = nullptr, double* gtheta = nullptr, const PfDev* pf = nullptr) {
    double* ws = (double*)g->ws;
    const int P = pr->P, H = pr->H, Ds = pr->dyn.E, D = pr->dyn.D, T = R * P;
    const size_t TD = (size_t)T * D, TDs = (size_t)T * Ds;
    const dim3 grid((P + PT_THREADS - 1) / PT_THREADS, R), cgrid((P + FS_WARPS - 1) / FS_WARPS, Ds, R);
    if (consistent && H > 1) cudaMemsetAsync(ws + L.G, 0, (size_t)H * (H + 1) / 2 * TDs * sizeof(double), st);
    PgDev b;
    static_cast<PtPolicy&>(b) = pt_policy(pr);
    b.eps = pf ? ws + L.fz : pr->eps; b.traj = pr->traj; b.step_risk = pr->step_risk;
    b.gx = ws + L.gx; b.gvar = ws + L.gvar; b.zbar = ws + L.zbar;
    FsBwd q;                                            // the cotangent rows G accumulate from zero
    q.P = P; q.T = T; q.H = H; q.D = D; q.Ds = Ds; q.np = pad64(pr->dyn.n); q.t = 0;
    q.ell = pr->dyn.ell; q.sf2 = pr->dyn.sf2;
    q.xh = ws + L.xt; q.Kh = ws + L.Kh; q.L = ws + L.L; q.eps = pr->eps;
    q.gx = b.gx; q.gvar = b.gvar; q.G = ws + L.G; q.A = ws + L.W; q.dir = ws + L.dir;
    const bool joint = pt_has_joint(pr);
    PjDev j = pj_dev(pr, R);
    j.xh = ws + L.xt; j.gxt = ws + L.gxt;
    PxBonus xb;
    if (bonus) {
        xb.P = P; xb.H = H; xb.E = Ds; xb.D = D; xb.t = 0; xb.n_rewards = pr->n_rewards;
        for (int k = 0; k < 8; ++k) xb.rewards[k] = k < pr->n_rewards ? pr->rewards[k] : pilco_reward_term();
        xb.traj = pr->traj; xb.tab = ws + L.tab; xb.gx = b.gx; xb.gxt = ws + L.gxt;
    }
    const PmChunks mc = pm_chunks(P);
    PmBwd mb;
    if (net) {                                          // the buffers' padding and the partials start at 0
        mb.net = *net; mb.Pp = mc.Pp; mb.RPp = (long long)R * mc.Pp;
        mb.in0 = ws + L.min0; mb.in1 = ws + L.min1; mb.in2 = ws + L.min2;
        mb.d1 = ws + L.md1; mb.d2 = ws + L.md2; mb.dout = ws + L.mdo;
        cudaMemsetAsync(ws + L.min0, 0, (L.mpart - L.min0) * sizeof(double), st);
        cudaMemsetAsync(ws + L.mpart, 0, (size_t)R * mc.nc * net->n_theta * sizeof(double), st);
    }
    if ((joint || bonus) && H > 0) {                    // x_bar_H = 0 and x~_bar_{H-1} = 0, then the joint terms' share
        cudaMemsetAsync(b.gx, 0, TDs * sizeof(double), st);
        cudaMemsetAsync(ws + L.gxt, 0, TD * sizeof(double), st);
    }
    for (int t = H - 1; t >= 0; --t) {
        b.t = t;
        if (sch) { b.W = pr->pol.W + t * sch->W_ts; b.b = pr->pol.b + t * sch->b_ts; }
        b.gxt = joint || bonus ? ws + L.gxt : nullptr;
        if (t < H - 1) {
            const double* xt = ws + L.xt + (size_t)t * TD;
            int rc;
            if (consistent) {
                q.t = t;
                launch_hi(fs_cond_bwd_kernel, cgrid, dim3(FS_WARPS * 32), 0, st, q);
                CUDA_LAUNCH_CHECK();
                rc = fs_vjp_launch(st, &pr->dyn, T, xt, b.gx, q.A, q.dir, ws + L.gxt, ws + L.vws);
            } else if (pf) {
                PfDev v = *pf;
                v.xh = xt; v.gmean = b.gx; v.gxt = ws + L.gxt;
                rc = pf_vjp_launch(st, v);
            } else {
                rc = pilco_gp_predict_vjp(&pr->dyn, T, xt, b.gx, b.gvar, ws + L.gxt, ws + L.vws, L.vws_bytes, st);
            }
            if (rc) return rc;
            b.gxt = ws + L.gxt;
        }
        if (joint) {
            j.t = t;
            launch_hi(pj_grad_kernel, grid, dim3(PT_THREADS), 0, st, j);
            CUDA_LAUNCH_CHECK();
        }
        if (bonus) {
            xb.t = t; xb.xh = ws + L.xt + (size_t)t * TD;
            if (const int rc = px_bonus_launch(st, grid, xb)) return rc;
        }
        b.var_prev = t > 0 ? ws + L.var + (size_t)(t - 1) * TDs : nullptr;
        if (nz) {
            PnBwd nb;
            static_cast<PgDev&>(nb) = b;
            nb.E = Ds; nb.tm = *tm; nb.phi = ws + L.phi; nb.phib = nullptr;
            nb.phiz = ws + L.phiz; nb.phibz = ws + L.phibz;
            if (const int rc = pn_reverse_launch(st, grid, nb)) return rc;
        } else if (tm) {
            PaBwd ab;
            static_cast<PgDev&>(ab) = b;
            ab.E = Ds; ab.tm = *tm; ab.phi = ws + L.phi; ab.phib = b.gxt ? ws + L.gxt : nullptr;
            if (const int rc = pa_reverse_launch(st, grid, ab)) return rc;
        } else if (net) {
            if (const int rc = pm_reverse_launch(st, grid, b, mb)) return rc;
            if (b.gxt) {                                // part[r, c] += d_l' [a_{l-1}; 1] over chunk c, layer by layer
                const int Dh = pr->pol.Ds, U = pr->pol.U, w1 = net->w1, w2 = net->w2, two = net->L == 2;
                const int wl = two ? w2 : w1;
                const int out[3] = {w1, w2, U}, n[3] = {Dh + 1, w1 + 1, wl + 1}, off[3] = {0, net->off2, net->offo};
                const double* dl[3] = {mb.d1, mb.d2, mb.dout};
                const double* in[3] = {mb.in0, mb.in1, two ? mb.in2 : mb.in1};
                for (int l = 0; l < 3; ++l) {
                    if (l == 1 && !two) continue;
                    const int rc = gemm(st, R * mc.nc, out[l], n[l], mc.Kc, 0, 1, 1.0, dl[l], (int)mb.RPp, mc.Kc,
                                        in[l], (int)mb.RPp, mc.Kc, 1.0, ws + L.mpart + off[l], n[l], net->n_theta);
                    if (rc) return rc;
                }
            }
        } else {
            launch_hi(pg_step_kernel, grid, dim3(PT_THREADS), 0, st, b);
            CUDA_LAUNCH_CHECK();
        }
        if (rs && t > 0) {
            PrBwd q;
            q.P = P; q.H = H; q.Ds = Ds; q.t = t; q.xi = rs->xi; q.eps = pr->eps;
            q.xp = ws + L.xp; q.mu = ws + L.rmu; q.L = ws + L.rL; q.var_prev = b.var_prev;
            q.gx = b.gx; q.gvar = b.gvar; q.sc = ws + L.rsc;
            if (const int rc = pr_reverse_launch(st, grid, q)) return rc;
        }
    }
    if (net) return pm_finish_launch(st, R, P, mc.nc, net->n_theta, ws + L.mpart, pr->ret, gtheta, g->value);
    return pg_reduce(pr, R, g, ws, L, st, nz ? ws + L.phiz : tm ? ws + L.phi : pr->traj, sch != nullptr);
}

// the moments kernel's arguments over the forward's traj and act (tm: the angles' map, or the identity)
static PxMom px_mom(const pilco_particles* pr, const TrigMap& tm, double b) {
    PxMom m;
    m.P = pr->P; m.H = pr->H; m.U = pr->pol.U; m.n_rewards = pr->n_rewards; m.tm = tm;
    m.traj = pr->traj; m.act = pr->act;
    for (int k = 0; k < 8; ++k) m.rewards[k] = k < pr->n_rewards ? pr->rewards[k] : pilco_reward_term();
    m.b = b; m.step_mean = m.step_var = m.sd = m.tab = nullptr;
    return m;
}

// The score-function gradient of R restarts after pt_forward(history) (DESIGN.md sections 16, 25):
//   ps_togo, ps_base, the cotangents of every step's predict and their VJPs, (joint terms) pj_grad over all H steps,
//   ps_zbar, pg_reduce
// Step-wise sampler: ps_cot, then the VJP of steps 0..H-2 in groups of whole steps.  The x~ history [H-1,T,D] and the
// cotangents [H-1,T,Ds] are contiguous, so a group of k steps is one VJP call at k T rows; a point's VJP does not
// depend on T or on its row, so the grouping changes no bit.
// Consistent sampler: pc_white_kernel (particles_cscore.cu) turns the weights into m_bar_t and v_bar_t, which stand
// where the pathwise sweep's x_bar_{t+1} and var_bar_t stand, then memset(Lambda) and [fs_cond_bwd<t>, fs_vjp<t> ->
// x~_bar_t] for t = H-2 .. 0.  Nothing chains x_bar between steps (x is held fixed), so there is no step kernel; Lambda
// accumulates over the steps, so the loop stays serial.
// Angles: the state-width cotangents are in E; ps_zbar and the reduction read the policy inputs from the phi history
// (Ds = Dh), and the joint terms' direct term starts at x~ column Dh.  Noise: the policy inputs are the phi(z)
// history; the VJPs act on x~, which holds phi(x), unchanged.  An active schedule: ps_zbar_sched and the per-step
// reduction in place of ps_zbar and pg_param (DESIGN.md section 28).
static int ps_run(const pilco_particles* pr, const PtOpt& o, const pilco_particles_grad* g, const PtWs& L,
                  cudaStream_t st) {
    double* ws = (double*)g->ws;
    const int R = o.R, P = pr->P, H = pr->H, Ds = pr->pol.Ds, E = pr->dyn.E, D = pr->dyn.D, T = R * P;
    const int nb = (P + PT_THREADS - 1) / PT_THREADS;
    const size_t TD = (size_t)T * D, TE = (size_t)T * E;
    const double* pin = o.noisy ? ws + L.phiz : o.mapped ? ws + L.phi : pr->traj;
    PsDev a;
    static_cast<PtPolicy&>(a) = pt_policy(pr);
    a.T = T;
    a.eps = pr->eps; a.traj = pin; a.step_reward = pr->step_reward; a.step_risk = pr->step_risk;
    a.var = o.consistent ? nullptr : ws + L.var; a.G = ws + L.togo; a.S = ws + L.gsum; a.gmean = ws + L.mw;
    a.gvar = ws + L.vw; a.gxt = ws + L.gxh; a.zbar = ws + L.zbar;
    a.direct = pt_has_joint(pr);
    if (H > 1) {
        launch_hi(ps_togo_kernel, dim3(nb, R), dim3(PT_THREADS), 0, st, a);
        CUDA_LAUNCH_CHECK();
        launch_hi(ps_base_kernel, dim3(H - 1, R), dim3(256), 0, st, a);
        CUDA_LAUNCH_CHECK();
        if (o.consistent) {
            PcWhite w;
            w.P = P; w.T = T; w.H = H; w.Ds = E;
            w.L = ws + L.L; w.eps = pr->eps; w.var = ws + L.var; w.G = a.G; w.S = a.S; w.mbar = a.gmean;
            w.vbar = a.gvar;
            if (const int rc = pc_white_launch(st, R, w)) return rc;
            cudaMemsetAsync(ws + L.G, 0, (size_t)H * (H + 1) / 2 * TE * sizeof(double), st);
            FsBwd q;                                    // as pg_reverse's; the cotangents come from the whitening reverse
            q.P = P; q.T = T; q.H = H; q.D = D; q.Ds = E; q.np = pad64(pr->dyn.n);
            q.ell = pr->dyn.ell; q.sf2 = pr->dyn.sf2;
            q.xh = ws + L.xt; q.Kh = ws + L.Kh; q.L = ws + L.L; q.eps = pr->eps;
            q.G = ws + L.G; q.A = ws + L.W; q.dir = ws + L.dir;
            const dim3 cgrid((P + FS_WARPS - 1) / FS_WARPS, E, R);
            for (int t = H - 2; t >= 0; --t) {
                q.t = t; q.gx = a.gmean + (size_t)t * TE; q.gvar = a.gvar + (size_t)t * TE;
                launch_hi(fs_cond_bwd_kernel, cgrid, dim3(FS_WARPS * 32), 0, st, q);
                CUDA_LAUNCH_CHECK();
                const int rc = fs_vjp_launch(st, &pr->dyn, T, ws + L.xt + (size_t)t * TD, q.gx, q.A, q.dir,
                                             ws + L.gxh + (size_t)t * TD, ws + L.vws);
                if (rc) return rc;
            }
        } else {
            PsDev ac = a;
            ac.Ds = E;
            launch_hi(ps_cot_kernel, dim3(nb * (H - 1), R), dim3(PT_THREADS), 0, st, ac);
            CUDA_LAUNCH_CHECK();
            const int grp = ps_group(T, H);
            for (int t0 = 0; t0 < H - 1; t0 += grp) {
                const int k = grp < H - 1 - t0 ? grp : H - 1 - t0;
                const size_t off = (size_t)t0 * T;
                const int rc = pilco_gp_predict_vjp(&pr->dyn, k * T, ws + L.xt + off * D, ws + L.mw + off * E,
                                                    ws + L.vw + off * E, ws + L.gxh + off * D, ws + L.vws, L.vws_bytes,
                                                    st);
                if (rc) return rc;
            }
        }
    }
    if (H > 0 && a.direct) {                            // the direct term: d v_k / d u_t of every step, on top of the VJP's
        cudaMemsetAsync(ws + L.gxh + (size_t)(H - 1) * TD, 0, TD * sizeof(double), st);
        PjDev j = pj_dev(pr, R);
        j.xh = ws + L.xt; j.gxt = ws + L.gxh; j.gstep = (long long)TD; j.first = Ds;
        launch_hi(pj_grad_kernel, dim3(nb * H, R), dim3(PT_THREADS), 0, st, j);
        CUDA_LAUNCH_CHECK();
    }
    if (H > 0 && o.sched) {                             // step t's W_t, b_t (DESIGN.md section 28)
        PsSched s;
        static_cast<PsDev&>(s) = a;
        s.W_ts = o.sch.W_ts; s.b_ts = o.sch.b_ts;
        launch_hi(ps_zbar_sched_kernel, dim3(nb * H, R), dim3(PT_THREADS), 0, st, s);
        CUDA_LAUNCH_CHECK();
    } else if (H > 0) {
        launch_hi(ps_zbar_kernel, dim3(nb * H, R), dim3(PT_THREADS), 0, st, a);
        CUDA_LAUNCH_CHECK();
    }
    return pg_reduce(pr, R, g, ws, L, st, pin, o.sched);
}

// ---- angular state dimensions (DESIGN.md section 20) ----------------------------------------------------------------
// The map of A >= 1 angles of the raw state (dyn.E dimensions) and the widths that go with it: PILCO_ERR_DIM for a
// repeated or out-of-range dimension, A > E, pol.Ds != E + A, dyn.D != pol.Ds + U, dyn.D > PILCO_MAX_D or an RBF
// policy whose input width is not pol.Ds.  pr is not NULL.
static int pa_map(const pilco_particles* pr, const pilco_angles* ang, TrigMap* tm) {
    const int E = pr->dyn.E, Dh = pr->pol.Ds;
    if (trig_map_make(E, ang->A, ang->dims, tm)) return PILCO_ERR_DIM;
    if (Dh != E + ang->A || pr->dyn.D != Dh + pr->pol.U || pr->dyn.D > MAXD) return PILCO_ERR_DIM;
    if (pr->pol.kind == PILCO_POLICY_RBF && pr->pol.rbf.D != Dh) return PILCO_ERR_DIM;
    return PILCO_OK;
}

static bool pa_none(const pilco_angles* ang) { return !ang || ang->A == 0; }

// ---- measurement noise at the policy's input (DESIGN.md section 23) -------------------------------------------------
// The noise's own checks, after the description's: PILCO_ERR_DIM for a non-finite or negative var[i] (i < dyn.E), then
// PILCO_ERR_NULL for nu == NULL with H > 0.  Fills n (sqrt(var), nu).  pr has passed its description's checks.
static int pn_noise(const pilco_particles* pr, const pilco_particles_noise* nz, PnNoise* n) {
    const int E = pr->dyn.E;
    for (int i = 0; i < MAXD; ++i) {
        const double v = i < E ? nz->v.var[i] : 0.0;
        if (!std::isfinite(v) || v < 0.0) return PILCO_ERR_DIM;
        n->sv[i] = std::sqrt(v);
    }
    if (!nz->nu && pr->H > 0) return PILCO_ERR_NULL;
    n->nu = nz->nu;
    return PILCO_OK;
}

// ---- exploration objective (DESIGN.md section 24) -------------------------------------------------------------------
// inactive (NULL, or b == 0 with step_var NULL): the call without exploration
static bool px_active(const pilco_exploration* ex) { return ex && (ex->b != 0.0 || ex->step_var); }

// the exploration's own checks, after the description's: PILCO_ERR_DIM for a non-finite b, PILCO_ERR_UNSUPPORTED for
// an ADD-channel box term (section 21's rule), PILCO_ERR_DIM for P < 2 (no sample variance).  pr is not NULL.
static int px_check(const pilco_particles* pr, const pilco_exploration* ex) {
    if (!std::isfinite(ex->b)) return PILCO_ERR_DIM;
    for (int k = 0; k < pr->n_rewards && k < 8; ++k)
        if (pr->rewards[k].channel == PILCO_CHANNEL_ADD && pr->rewards[k].kind == PILCO_REWARD_BOX)
            return PILCO_ERR_UNSUPPORTED;
    if (pr->P < 2) return PILCO_ERR_DIM;
    return PILCO_OK;
}

// ---- time-varying linear policy (DESIGN.md section 28) ----------------------------------------------------------------
// active: sch not NULL and a non-zero stride; an inactive schedule is the call without it
static bool pt_sched_active(const pilco_policy_schedule* sch) { return sch && (sch->W_ts != 0 || sch->b_ts != 0); }

// ---- one validator, one query, one call path --------------------------------------------------------------------------
// Everything a call checks before its workspace, in this order: NULL pr, the angles' map (A != 0), the description
// (the policy's batch strides as o->batched allows), R, the gradient's outputs (a batched forward's: value), the
// noise, the exploration (active only).  Each family's call is the most general call with NULL for the features it
// lacks, so ang == NULL or A == 0 is the call without angles, nz == NULL the call without noise and an inactive ex the
// call without exploration.
// Resampled calls (o->resampled, no angles, noise or exploration), after the gradient's outputs: PILCO_ERR_NULL for rs
// NULL or xi NULL with H > 0, then PILCO_ERR_DIM for P < 2 (no sample covariance).
// Scheduled calls (DESIGN.md section 28), after everything else: PILCO_ERR_DIM for a negative stride, then
// PILCO_ERR_UNSUPPORTED for an active schedule with an RBF policy.  sch NULL or both strides 0 is the call without it.
// MLP calls (o->mlp, DESIGN.md section 29; no angles, noise or schedule): the description's policy checks are the
// MLP's (pt_check_desc), and the gradient's outputs are value, ws and mlp->gtheta.
// Feature calls (o->features, DESIGN.md section 30; no refit, schedule or score estimator): pr->eps is not checked,
// and after everything else PILCO_ERR_NULL for fd, omega, w or v NULL, then PILCO_ERR_DIM for F out of range.
static bool pf_F_ok(int F) { return F >= 1 && F <= PILCO_MAX_FEATURES; }

static int pt_validate(PtOpt* o, const pilco_particles* pr, const pilco_angles* ang, const pilco_particles_noise* nz,
                       const pilco_exploration* ex, int R, const pilco_particles_grad* g,
                       const pilco_particles_resample* rs = nullptr, const pilco_policy_schedule* sch = nullptr,
                       const pilco_mlp* mlp = nullptr, const pilco_feature_draws* fd = nullptr) {
    if (!pr) return PILCO_ERR_NULL;
    const bool angles = !pa_none(ang);
    if (angles)
        if (const int rc = pa_map(pr, ang, &o->tm)) return rc;
    if (const int rc = pt_check_desc(pr, o->batched, angles ? o->tm.A : 0, o->mlp, mlp, !o->features)) return rc;
    if (!pt_batch_ok(pr->P, R)) return PILCO_ERR_DIM;   // the unbatched calls' R = 1 passes with the description
    if (o->call != PT_FORWARD) {
        if (const int rc = pg_check(pr, g, o->mlp ? mlp : nullptr)) return rc;
    } else if (o->batched && !o->value) return PILCO_ERR_NULL;
    if (o->mlp) o->net = pm_net(pr, mlp);
    if (o->resampled) {
        if (!rs || (!rs->xi && pr->H > 0)) return PILCO_ERR_NULL;
        if (pr->P < 2) return PILCO_ERR_DIM;
        o->rs = *rs;
    }
    if (!angles) trig_map_make(pr->dyn.E, 0, nullptr, &o->tm);     // 1 <= E <= PILCO_MAX_E once the description passed
    if (nz)
        if (const int rc = pn_noise(pr, nz, &o->nz)) return rc;
    o->explore = px_active(ex);
    if (o->explore) {
        if (const int rc = px_check(pr, ex)) return rc;
        o->b = ex->b; o->step_var = ex->step_var; o->bonus = ex->b != 0.0;
    }
    o->R = R; o->mapped = angles || nz; o->noisy = nz != nullptr;
    if (sch && (sch->W_ts < 0 || sch->b_ts < 0)) return PILCO_ERR_DIM;
    o->sched = pt_sched_active(sch);
    if (o->sched) {
        if (pt_rbf(pr)) return PILCO_ERR_UNSUPPORTED;
        o->sch = *sch;
    }
    if (o->features) {
        if (!fd || !fd->omega || !fd->w || !fd->v) return PILCO_ERR_NULL;
        if (!pf_F_ok(fd->F)) return PILCO_ERR_DIM;
        o->fd = *fd;
    }
    return PILCO_OK;
}

// A call's workspace: its layout's total, 0 where the call would fail on its sizes.  The sizes accepted are the
// description's own (pt_sizes_ok, not its width consistency), R, the angles' map, 1 <= E <= PILCO_MAX_E and valid
// variances with noise, and the exploration's checks when active; a schedule only adds non-negative strides (its
// workspace is the call's without it); an MLP call adds mlp != NULL and its sizes (L, the widths); a feature call fd !=
// NULL and F in range.
static size_t pt_query(PtOpt o, const pilco_particles* pr, const pilco_angles* ang, const pilco_particles_noise* nz,
                       const pilco_exploration* ex, int R, const pilco_policy_schedule* sch = nullptr,
                       const pilco_mlp* mlp = nullptr, const pilco_feature_draws* fd = nullptr) {
    if (!pr || !pt_sizes_ok(pr) || !pt_batch_ok(pr->P, R)) return 0;
    if (o.features && (!fd || !pf_F_ok(fd->F))) return 0;
    if (o.mlp) {                                        // the MLP's sizes (NULL: none to size the workspace with)
        if (!mlp || !pm_sizes_ok(mlp)) return 0;
        o.net = pm_net(pr, mlp);
    }
    if (sch && (sch->W_ts < 0 || sch->b_ts < 0)) return 0;
    if (!pa_none(ang) && pa_map(pr, ang, &o.tm)) return 0;
    if (nz && (pr->dyn.E < 1 || pr->dyn.E > MAXE || pn_noise(pr, nz, &o.nz))) return 0;
    o.explore = px_active(ex);
    if (o.explore && px_check(pr, ex)) return 0;
    if (o.resampled && pr->P < 2) return 0;
    o.R = R; o.mapped = nz || !pa_none(ang); o.noisy = nz != nullptr;
    return pt_layout(pr, o).total;
}

// Every rollout call: validate, lay out, check the workspace (pr's for the forward, g's for a gradient), prepare, then
// the forward (with its history for a gradient) and the gradient's reverse part.  Pathwise with exploration: the
// moments after the forward; with b != 0 the bonus's share in the reverse sweep and the bonus in value after it.
static int pt_call(PtOpt o, const pilco_particles* pr, const pilco_angles* ang, const pilco_particles_noise* nz,
                   const pilco_exploration* ex, int R, const pilco_particles_grad* g, pilco_stream_t stream,
                   const pilco_particles_resample* rs = nullptr, const pilco_policy_schedule* sch = nullptr,
                   const pilco_mlp* mlp = nullptr, const pilco_feature_draws* fd = nullptr) {
    if (const int rc = pt_validate(&o, pr, ang, nz, ex, R, g, rs, sch, mlp, fd)) return rc;
    const bool fwd = o.call == PT_FORWARD;
    const PtWs L = pt_layout(pr, o);
    if (const int rc = fwd ? pt_check_ws(pr->ws, pr->ws_bytes, L.total) : pt_check_ws(g->ws, g->ws_bytes, L.total))
        return rc;
    if (o.consistent) {
        if (const int rc = fs_predict_prepare()) return rc;
        if (!fwd)
            if (const int rc = fs_vjp_prepare()) return rc;
    }
    cudaStream_t st = (cudaStream_t)stream;
    double* ws = (double*)(fwd ? pr->ws : g->ws);
    const TrigMap* tm = o.mapped ? &o.tm : nullptr;
    const PnNoise* n = o.noisy ? &o.nz : nullptr;
    const pilco_particles_resample* rsv = o.resampled ? &o.rs : nullptr;
    const pilco_policy_schedule* sv = o.sched ? &o.sch : nullptr;
    const PmNet* net = o.mlp ? &o.net : nullptr;
    PfDev q = {};
    if (o.features) {
        q.T = (long long)R * pr->P; q.P = pr->P; q.D = pr->dyn.D; q.E = pr->dyn.E; q.F = o.fd.F; q.n = pr->dyn.n;
        q.omega = o.fd.omega; q.X = pr->dyn.X; q.ell = pr->dyn.ell; q.sf2 = pr->dyn.sf2; q.w = o.fd.w; q.v = o.fd.v;
    }
    const PfDev* pf = o.features ? &q : nullptr;
    if (const int rc = pt_forward(pr, R, ws, L, o.consistent, !fwd, st, tm, n, rsv, sv, net, pf)) return rc;
    // a batched forward's value: pm_finish_kernel with no parameters is its value CTA alone, the same fixed-order mean
    // as pg_param_kernel's and pg_sched_kernel's
    if (fwd) return o.batched ? pm_finish_launch(st, R, pr->P, 0, 0, nullptr, pr->ret, nullptr, o.value) : PILCO_OK;
    if (o.call == PT_SCORE) return ps_run(pr, o, g, L, st);
    if (o.explore) {
        PxMom m = px_mom(pr, o.tm, o.b);
        m.step_var = o.step_var; m.sd = ws + L.sd; m.tab = o.bonus ? ws + L.tab : nullptr;
        if (const int rc = px_moments_launch(st, R, m)) return rc;
    }
    if (const int rc = pg_reverse(pr, R, g, L, o.consistent, st, tm, n, o.bonus, rsv, sv, net,
                                  o.mlp ? mlp->gtheta : nullptr, pf))
        return rc;
    if (o.bonus && pr->H > 0) return px_value_launch(st, R, pr->H, o.b, ws + L.sd, g->value);
    return PILCO_OK;
}

// the sampler, the call and whether the policy's batch strides are honoured, per family
static const PtOpt FWD = {false, PT_FORWARD, false}, CFWD = {true, PT_FORWARD, false};
static const PtOpt PATH1 = {false, PT_PATHWISE, false}, PATH = {false, PT_PATHWISE, true};
static const PtOpt CPATH = {true, PT_PATHWISE, true}, SCORE = {false, PT_SCORE, true}, CSCORE = {true, PT_SCORE, true};
static const PtOpt RFWD = {false, PT_FORWARD, false, true}, RPATH = {false, PT_PATHWISE, true, true};
static const PtOpt BFWD = {false, PT_FORWARD, true}, CBFWD = {true, PT_FORWARD, true};

// the MLP calls (DESIGN.md section 29): a family's options with o.mlp
static PtOpt pm_opt(PtOpt o) { o.mlp = true; return o; }

// the feature calls (DESIGN.md section 30): the step-wise forward and pathwise options with o.features
static PtOpt pf_opt(PtOpt o) { o.features = true; return o; }

extern "C" {

size_t pilco_particles_workspace_bytes(const pilco_particles* pr) {
    return pt_query(FWD, pr, nullptr, nullptr, nullptr, 1);
}

int pilco_particles_rollout(const pilco_particles* pr, pilco_stream_t stream) {
    return pt_call(FWD, pr, nullptr, nullptr, nullptr, 1, nullptr, stream);
}

size_t pilco_particles_grad_workspace_bytes(const pilco_particles* pr) {
    return pt_query(PATH1, pr, nullptr, nullptr, nullptr, 1);
}

int pilco_particles_rollout_grad(const pilco_particles* pr, const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(PATH1, pr, nullptr, nullptr, nullptr, 1, g, stream);
}

size_t pilco_particles_batch_grad_workspace_bytes(const pilco_particles* pr, int R) {
    return pt_query(PATH, pr, nullptr, nullptr, nullptr, R);
}

int pilco_particles_rollout_batch_grad(const pilco_particles* pr, int R, const pilco_particles_grad* g,
                                       pilco_stream_t stream) {
    return pt_call(PATH, pr, nullptr, nullptr, nullptr, R, g, stream);
}

size_t pilco_particles_consistent_workspace_bytes(const pilco_particles* pr) {
    return pt_query(CFWD, pr, nullptr, nullptr, nullptr, 1);
}

int pilco_particles_rollout_consistent(const pilco_particles* pr, pilco_stream_t stream) {
    return pt_call(CFWD, pr, nullptr, nullptr, nullptr, 1, nullptr, stream);
}

size_t pilco_particles_consistent_grad_workspace_bytes(const pilco_particles* pr, int R) {
    return pt_query(CPATH, pr, nullptr, nullptr, nullptr, R);
}

int pilco_particles_rollout_consistent_grad(const pilco_particles* pr, int R, const pilco_particles_grad* g,
                                            pilco_stream_t stream) {
    return pt_call(CPATH, pr, nullptr, nullptr, nullptr, R, g, stream);
}

size_t pilco_particles_score_grad_workspace_bytes(const pilco_particles* pr, int R) {
    return pt_query(SCORE, pr, nullptr, nullptr, nullptr, R);
}

int pilco_particles_rollout_score_grad(const pilco_particles* pr, int R, const pilco_particles_grad* g,
                                       pilco_stream_t stream) {
    return pt_call(SCORE, pr, nullptr, nullptr, nullptr, R, g, stream);
}

size_t pilco_particles_angles_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang) {
    return pt_query(FWD, pr, ang, nullptr, nullptr, 1);
}

int pilco_particles_angles_rollout(const pilco_particles* pr, const pilco_angles* ang, pilco_stream_t stream) {
    return pt_call(FWD, pr, ang, nullptr, nullptr, 1, nullptr, stream);
}

size_t pilco_particles_angles_consistent_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang) {
    return pt_query(CFWD, pr, ang, nullptr, nullptr, 1);
}

int pilco_particles_angles_consistent_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                              pilco_stream_t stream) {
    return pt_call(CFWD, pr, ang, nullptr, nullptr, 1, nullptr, stream);
}

size_t pilco_particles_angles_batch_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang, int R) {
    return pt_query(PATH, pr, ang, nullptr, nullptr, R);
}

int pilco_particles_angles_batch_grad_rollout(const pilco_particles* pr, const pilco_angles* ang, int R,
                                              const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(PATH, pr, ang, nullptr, nullptr, R, g, stream);
}

size_t pilco_particles_angles_consistent_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                              int R) {
    return pt_query(CPATH, pr, ang, nullptr, nullptr, R);
}

int pilco_particles_angles_consistent_grad_rollout(const pilco_particles* pr, const pilco_angles* ang, int R,
                                                   const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(CPATH, pr, ang, nullptr, nullptr, R, g, stream);
}

size_t pilco_particles_angles_score_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang, int R) {
    return pt_query(SCORE, pr, ang, nullptr, nullptr, R);
}

int pilco_particles_angles_score_grad_rollout(const pilco_particles* pr, const pilco_angles* ang, int R,
                                              const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(SCORE, pr, ang, nullptr, nullptr, R, g, stream);
}

size_t pilco_particles_noisy_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                             const pilco_particles_noise* nz) {
    return pt_query(FWD, pr, ang, nz, nullptr, 1);
}

int pilco_particles_noisy_rollout(const pilco_particles* pr, const pilco_angles* ang, const pilco_particles_noise* nz,
                                  pilco_stream_t stream) {
    return pt_call(FWD, pr, ang, nz, nullptr, 1, nullptr, stream);
}

size_t pilco_particles_noisy_consistent_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                        const pilco_particles_noise* nz) {
    return pt_query(CFWD, pr, ang, nz, nullptr, 1);
}

int pilco_particles_noisy_consistent_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                             const pilco_particles_noise* nz, pilco_stream_t stream) {
    return pt_call(CFWD, pr, ang, nz, nullptr, 1, nullptr, stream);
}

size_t pilco_particles_noisy_batch_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                        const pilco_particles_noise* nz, int R) {
    return pt_query(PATH, pr, ang, nz, nullptr, R);
}

int pilco_particles_noisy_batch_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                             const pilco_particles_noise* nz, int R, const pilco_particles_grad* g,
                                             pilco_stream_t stream) {
    return pt_call(PATH, pr, ang, nz, nullptr, R, g, stream);
}

size_t pilco_particles_noisy_consistent_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                             const pilco_particles_noise* nz, int R) {
    return pt_query(CPATH, pr, ang, nz, nullptr, R);
}

int pilco_particles_noisy_consistent_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                  const pilco_particles_noise* nz, int R,
                                                  const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(CPATH, pr, ang, nz, nullptr, R, g, stream);
}

size_t pilco_particles_noisy_score_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                        const pilco_particles_noise* nz, int R) {
    return pt_query(SCORE, pr, ang, nz, nullptr, R);
}

int pilco_particles_noisy_score_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                             const pilco_particles_noise* nz, int R, const pilco_particles_grad* g,
                                             pilco_stream_t stream) {
    return pt_call(SCORE, pr, ang, nz, nullptr, R, g, stream);
}

size_t pilco_particles_explore_batch_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                          const pilco_particles_noise* nz, const pilco_exploration* ex,
                                                          int R) {
    return pt_query(PATH, pr, ang, nz, ex, R);
}

int pilco_particles_explore_batch_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                               const pilco_particles_noise* nz, const pilco_exploration* ex, int R,
                                               const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(PATH, pr, ang, nz, ex, R, g, stream);
}

size_t pilco_particles_explore_consistent_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                               const pilco_particles_noise* nz,
                                                               const pilco_exploration* ex, int R) {
    return pt_query(CPATH, pr, ang, nz, ex, R);
}

int pilco_particles_explore_consistent_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                    const pilco_particles_noise* nz, const pilco_exploration* ex, int R,
                                                    const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(CPATH, pr, ang, nz, ex, R, g, stream);
}

size_t pilco_particles_consistent_score_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                             const pilco_particles_noise* nz, int R) {
    return pt_query(CSCORE, pr, ang, nz, nullptr, R);
}

int pilco_particles_consistent_score_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                  const pilco_particles_noise* nz, int R,
                                                  const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(CSCORE, pr, ang, nz, nullptr, R, g, stream);
}

size_t pilco_particles_resampled_workspace_bytes(const pilco_particles* pr, const pilco_particles_resample* rs) {
    (void)rs;                                           // the sizes do not depend on it
    return pt_query(RFWD, pr, nullptr, nullptr, nullptr, 1);
}

int pilco_particles_resampled_rollout(const pilco_particles* pr, const pilco_particles_resample* rs,
                                      pilco_stream_t stream) {
    return pt_call(RFWD, pr, nullptr, nullptr, nullptr, 1, nullptr, stream, rs);
}

size_t pilco_particles_resampled_grad_workspace_bytes(const pilco_particles* pr, const pilco_particles_resample* rs,
                                                      int R) {
    (void)rs;
    return pt_query(RPATH, pr, nullptr, nullptr, nullptr, R);
}

int pilco_particles_resampled_grad_rollout(const pilco_particles* pr, const pilco_particles_resample* rs, int R,
                                           const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(RPATH, pr, nullptr, nullptr, nullptr, R, g, stream, rs);
}

// time-varying linear policy (DESIGN.md section 28): each family's most general call with sch
size_t pilco_particles_scheduled_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                 const pilco_particles_noise* nz, const pilco_policy_schedule* sch) {
    return pt_query(FWD, pr, ang, nz, nullptr, 1, sch);
}

int pilco_particles_scheduled_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                      const pilco_particles_noise* nz, const pilco_policy_schedule* sch,
                                      pilco_stream_t stream) {
    return pt_call(FWD, pr, ang, nz, nullptr, 1, nullptr, stream, nullptr, sch);
}

size_t pilco_particles_scheduled_consistent_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                            const pilco_particles_noise* nz,
                                                            const pilco_policy_schedule* sch) {
    return pt_query(CFWD, pr, ang, nz, nullptr, 1, sch);
}

int pilco_particles_scheduled_consistent_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                 const pilco_particles_noise* nz, const pilco_policy_schedule* sch,
                                                 pilco_stream_t stream) {
    return pt_call(CFWD, pr, ang, nz, nullptr, 1, nullptr, stream, nullptr, sch);
}

size_t pilco_particles_scheduled_batch_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                            const pilco_particles_noise* nz,
                                                            const pilco_exploration* ex,
                                                            const pilco_policy_schedule* sch, int R) {
    return pt_query(PATH, pr, ang, nz, ex, R, sch);
}

int pilco_particles_scheduled_batch_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                 const pilco_particles_noise* nz, const pilco_exploration* ex,
                                                 const pilco_policy_schedule* sch, int R,
                                                 const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(PATH, pr, ang, nz, ex, R, g, stream, nullptr, sch);
}

// batched forward-only rollouts (DESIGN.md section 31): the scheduled gradient calls' forward without their histories
size_t pilco_particles_scheduled_batch_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                       const pilco_particles_noise* nz,
                                                       const pilco_policy_schedule* sch, int R) {
    return pt_query(BFWD, pr, ang, nz, nullptr, R, sch);
}

int pilco_particles_scheduled_batch_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                            const pilco_particles_noise* nz, const pilco_policy_schedule* sch, int R,
                                            double* value, pilco_stream_t stream) {
    PtOpt o = BFWD;
    o.value = value;
    return pt_call(o, pr, ang, nz, nullptr, R, nullptr, stream, nullptr, sch);
}

size_t pilco_particles_scheduled_consistent_batch_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                                  const pilco_particles_noise* nz,
                                                                  const pilco_policy_schedule* sch, int R) {
    return pt_query(CBFWD, pr, ang, nz, nullptr, R, sch);
}

int pilco_particles_scheduled_consistent_batch_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                       const pilco_particles_noise* nz,
                                                       const pilco_policy_schedule* sch, int R, double* value,
                                                       pilco_stream_t stream) {
    PtOpt o = CBFWD;
    o.value = value;
    return pt_call(o, pr, ang, nz, nullptr, R, nullptr, stream, nullptr, sch);
}

// batched forward-only rollouts of stationary policies (DESIGN.md section 33): the explore gradient calls' forward
// (ex NULL) without their histories; the same options as section 31's with no schedule
size_t pilco_particles_batch_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                             const pilco_particles_noise* nz, int R) {
    return pt_query(BFWD, pr, ang, nz, nullptr, R);
}

int pilco_particles_batch_rollout(const pilco_particles* pr, const pilco_angles* ang, const pilco_particles_noise* nz,
                                  int R, double* value, pilco_stream_t stream) {
    PtOpt o = BFWD;
    o.value = value;
    return pt_call(o, pr, ang, nz, nullptr, R, nullptr, stream);
}

size_t pilco_particles_consistent_batch_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                        const pilco_particles_noise* nz, int R) {
    return pt_query(CBFWD, pr, ang, nz, nullptr, R);
}

int pilco_particles_consistent_batch_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                             const pilco_particles_noise* nz, int R, double* value,
                                             pilco_stream_t stream) {
    PtOpt o = CBFWD;
    o.value = value;
    return pt_call(o, pr, ang, nz, nullptr, R, nullptr, stream);
}

size_t pilco_particles_scheduled_consistent_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                                 const pilco_particles_noise* nz,
                                                                 const pilco_exploration* ex,
                                                                 const pilco_policy_schedule* sch, int R) {
    return pt_query(CPATH, pr, ang, nz, ex, R, sch);
}

int pilco_particles_scheduled_consistent_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                      const pilco_particles_noise* nz, const pilco_exploration* ex,
                                                      const pilco_policy_schedule* sch, int R,
                                                      const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(CPATH, pr, ang, nz, ex, R, g, stream, nullptr, sch);
}

size_t pilco_particles_scheduled_score_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                            const pilco_particles_noise* nz,
                                                            const pilco_policy_schedule* sch, int R) {
    return pt_query(SCORE, pr, ang, nz, nullptr, R, sch);
}

int pilco_particles_scheduled_score_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                 const pilco_particles_noise* nz, const pilco_policy_schedule* sch,
                                                 int R, const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(SCORE, pr, ang, nz, nullptr, R, g, stream, nullptr, sch);
}

size_t pilco_particles_scheduled_consistent_score_grad_workspace_bytes(const pilco_particles* pr,
                                                                       const pilco_angles* ang,
                                                                       const pilco_particles_noise* nz,
                                                                       const pilco_policy_schedule* sch, int R) {
    return pt_query(CSCORE, pr, ang, nz, nullptr, R, sch);
}

int pilco_particles_scheduled_consistent_score_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                                            const pilco_particles_noise* nz,
                                                            const pilco_policy_schedule* sch, int R,
                                                            const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(CSCORE, pr, ang, nz, nullptr, R, g, stream, nullptr, sch);
}

size_t pilco_particles_scheduled_resampled_workspace_bytes(const pilco_particles* pr,
                                                           const pilco_particles_resample* rs,
                                                           const pilco_policy_schedule* sch) {
    (void)rs;
    return pt_query(RFWD, pr, nullptr, nullptr, nullptr, 1, sch);
}

int pilco_particles_scheduled_resampled_rollout(const pilco_particles* pr, const pilco_particles_resample* rs,
                                                const pilco_policy_schedule* sch, pilco_stream_t stream) {
    return pt_call(RFWD, pr, nullptr, nullptr, nullptr, 1, nullptr, stream, rs, sch);
}

size_t pilco_particles_scheduled_resampled_grad_workspace_bytes(const pilco_particles* pr,
                                                                const pilco_particles_resample* rs,
                                                                const pilco_policy_schedule* sch, int R) {
    (void)rs;
    return pt_query(RPATH, pr, nullptr, nullptr, nullptr, R, sch);
}

int pilco_particles_scheduled_resampled_grad_rollout(const pilco_particles* pr, const pilco_particles_resample* rs,
                                                     const pilco_policy_schedule* sch, int R,
                                                     const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(RPATH, pr, nullptr, nullptr, nullptr, R, g, stream, rs, sch);
}

// tanh MLP policies (DESIGN.md section 29): the step-wise, consistent and resampled samplers, forward and pathwise
size_t pilco_particles_mlp_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp) {
    return pt_query(pm_opt(FWD), pr, nullptr, nullptr, nullptr, 1, nullptr, mlp);
}

int pilco_particles_mlp_rollout(const pilco_particles* pr, const pilco_mlp* mlp, pilco_stream_t stream) {
    return pt_call(pm_opt(FWD), pr, nullptr, nullptr, nullptr, 1, nullptr, stream, nullptr, nullptr, mlp);
}

size_t pilco_particles_mlp_consistent_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp) {
    return pt_query(pm_opt(CFWD), pr, nullptr, nullptr, nullptr, 1, nullptr, mlp);
}

int pilco_particles_mlp_consistent_rollout(const pilco_particles* pr, const pilco_mlp* mlp, pilco_stream_t stream) {
    return pt_call(pm_opt(CFWD), pr, nullptr, nullptr, nullptr, 1, nullptr, stream, nullptr, nullptr, mlp);
}

size_t pilco_particles_mlp_resampled_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                     const pilco_particles_resample* rs) {
    (void)rs;                                           // the sizes do not depend on it
    return pt_query(pm_opt(RFWD), pr, nullptr, nullptr, nullptr, 1, nullptr, mlp);
}

int pilco_particles_mlp_resampled_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                          const pilco_particles_resample* rs, pilco_stream_t stream) {
    return pt_call(pm_opt(RFWD), pr, nullptr, nullptr, nullptr, 1, nullptr, stream, rs, nullptr, mlp);
}

size_t pilco_particles_mlp_batch_grad_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                      const pilco_exploration* ex, int R) {
    return pt_query(pm_opt(PATH), pr, nullptr, nullptr, ex, R, nullptr, mlp);
}

int pilco_particles_mlp_batch_grad_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                           const pilco_exploration* ex, int R, const pilco_particles_grad* g,
                                           pilco_stream_t stream) {
    return pt_call(pm_opt(PATH), pr, nullptr, nullptr, ex, R, g, stream, nullptr, nullptr, mlp);
}

size_t pilco_particles_mlp_consistent_grad_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                           const pilco_exploration* ex, int R) {
    return pt_query(pm_opt(CPATH), pr, nullptr, nullptr, ex, R, nullptr, mlp);
}

int pilco_particles_mlp_consistent_grad_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                                const pilco_exploration* ex, int R, const pilco_particles_grad* g,
                                                pilco_stream_t stream) {
    return pt_call(pm_opt(CPATH), pr, nullptr, nullptr, ex, R, g, stream, nullptr, nullptr, mlp);
}

size_t pilco_particles_mlp_resampled_grad_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                          const pilco_particles_resample* rs, int R) {
    (void)rs;
    return pt_query(pm_opt(RPATH), pr, nullptr, nullptr, nullptr, R, nullptr, mlp);
}

int pilco_particles_mlp_resampled_grad_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                               const pilco_particles_resample* rs, int R,
                                               const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(pm_opt(RPATH), pr, nullptr, nullptr, nullptr, R, g, stream, rs, nullptr, mlp);
}

// batched forward-only MLP rollouts (DESIGN.md section 33): the MLP gradient calls' forward (ex NULL)
size_t pilco_particles_mlp_batch_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp, int R) {
    return pt_query(pm_opt(BFWD), pr, nullptr, nullptr, nullptr, R, nullptr, mlp);
}

int pilco_particles_mlp_batch_rollout(const pilco_particles* pr, const pilco_mlp* mlp, int R, double* value,
                                      pilco_stream_t stream) {
    PtOpt o = pm_opt(BFWD);
    o.value = value;
    return pt_call(o, pr, nullptr, nullptr, nullptr, R, nullptr, stream, nullptr, nullptr, mlp);
}

size_t pilco_particles_mlp_consistent_batch_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp, int R) {
    return pt_query(pm_opt(CBFWD), pr, nullptr, nullptr, nullptr, R, nullptr, mlp);
}

int pilco_particles_mlp_consistent_batch_rollout(const pilco_particles* pr, const pilco_mlp* mlp, int R, double* value,
                                                 pilco_stream_t stream) {
    PtOpt o = pm_opt(CBFWD);
    o.value = value;
    return pt_call(o, pr, nullptr, nullptr, nullptr, R, nullptr, stream, nullptr, nullptr, mlp);
}

// function samples from random-feature draws (DESIGN.md section 30); the draw call is in particles_features.cu
size_t pilco_particles_features_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                const pilco_particles_noise* nz, const pilco_feature_draws* fd) {
    return pt_query(pf_opt(FWD), pr, ang, nz, nullptr, 1, nullptr, nullptr, fd);
}

int pilco_particles_features_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                     const pilco_particles_noise* nz, const pilco_feature_draws* fd,
                                     pilco_stream_t stream) {
    return pt_call(pf_opt(FWD), pr, ang, nz, nullptr, 1, nullptr, stream, nullptr, nullptr, nullptr, fd);
}

size_t pilco_particles_features_grad_workspace_bytes(const pilco_particles* pr, const pilco_angles* ang,
                                                     const pilco_particles_noise* nz, const pilco_exploration* ex,
                                                     const pilco_feature_draws* fd, int R) {
    return pt_query(pf_opt(PATH), pr, ang, nz, ex, R, nullptr, nullptr, fd);
}

int pilco_particles_features_grad_rollout(const pilco_particles* pr, const pilco_angles* ang,
                                          const pilco_particles_noise* nz, const pilco_exploration* ex,
                                          const pilco_feature_draws* fd, int R, const pilco_particles_grad* g,
                                          pilco_stream_t stream) {
    return pt_call(pf_opt(PATH), pr, ang, nz, ex, R, g, stream, nullptr, nullptr, nullptr, fd);
}

size_t pilco_particles_mlp_features_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                    const pilco_feature_draws* fd) {
    return pt_query(pf_opt(pm_opt(FWD)), pr, nullptr, nullptr, nullptr, 1, nullptr, mlp, fd);
}

int pilco_particles_mlp_features_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                         const pilco_feature_draws* fd, pilco_stream_t stream) {
    return pt_call(pf_opt(pm_opt(FWD)), pr, nullptr, nullptr, nullptr, 1, nullptr, stream, nullptr, nullptr, mlp, fd);
}

size_t pilco_particles_mlp_features_grad_workspace_bytes(const pilco_particles* pr, const pilco_mlp* mlp,
                                                         const pilco_exploration* ex, const pilco_feature_draws* fd,
                                                         int R) {
    return pt_query(pf_opt(pm_opt(PATH)), pr, nullptr, nullptr, ex, R, nullptr, mlp, fd);
}

int pilco_particles_mlp_features_grad_rollout(const pilco_particles* pr, const pilco_mlp* mlp,
                                              const pilco_exploration* ex, const pilco_feature_draws* fd, int R,
                                              const pilco_particles_grad* g, pilco_stream_t stream) {
    return pt_call(pf_opt(pm_opt(PATH)), pr, nullptr, nullptr, ex, R, g, stream, nullptr, nullptr, mlp, fd);
}

int pilco_particles_reward_moments(const pilco_particles* pr, const pilco_angles* ang, int R, double* step_mean,
                                   double* step_var, pilco_stream_t stream) {
    if (!pr) return PILCO_ERR_NULL;
    const int E = pr->dyn.E, U = pr->pol.U;
    TrigMap tm;
    const int A = pa_none(ang) ? 0 : ang->A;
    if (pr->P < 2 || pr->H < 0 || R < 1 || R > 65535 || U < 1 || trig_map_make(E, A, A ? ang->dims : nullptr, &tm) ||
        E > MAXE || pr->pol.Ds != E + A || E + A + U > MAXD)
        return PILCO_ERR_DIM;
    if (const int rc = pt_check_rewards(pr, true)) return rc;
    if (pr->H > 0 && (!pr->traj || !pr->act)) return PILCO_ERR_NULL;
    PxMom m = px_mom(pr, tm, 0.0);
    m.step_mean = step_mean; m.step_var = step_var;
    return px_moments_launch((cudaStream_t)stream, R, m);
}

}  // extern "C"
