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
#include <initializer_list>
#include "common.cuh"
#include "risk_math.cuh"

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

// ---- reverse sweep of pilco_particles_rollout_grad (DESIGN.md section 12) ---------------------------------------------
// Per particle, x_bar_H = 0 and t = H-1 .. 0 (s_t = sqrt(max(var_t, 0)), z_t the pre-squash action):
//   mu_bar_t = x_bar_{t+1},  var_bar_t = x_bar_{t+1} o eps_t / (2 s_t) where var_t > 0, else 0
//   x~_bar_t = pilco_gp_predict_vjp at x~_t;  z_bar_t = x~_bar_t[Ds:] o maxa e^{-su/2} cos(z_t)  (when squashed)
//   x_bar_t  = x_bar_{t+1} + x~_bar_t[:Ds] + (d pi / dx)' z_bar_t + sum_k a_kt grad v_k(x_t)
// a_kt = coef_k (ADD) or coef_k mult_mu prod_{s != t} (1 - risk_s) (MULT).  x_H carries no reward, so the sweep
// starts at t = H-1 with x_bar_H = 0 and x~_bar_{H-1} = 0: H-1 VJP calls.
struct PgDev : PtPolicy {
    int t;
    const double* eps; const double* traj; const double* step_risk;
    const double* gxt;          // VJP of step t at x~_t [R P,D]; NULL at t = H-1
    const double* var_prev;     // var_{t-1} [R P,Ds] (t > 0)
    double* gx;                 // [R P,Ds] x_bar_{t+1} in, x_bar_t out (= the gmean of step t-1's VJP)
    double* gvar;               // [R P,Ds] the gvar of step t-1's VJP
    double* zbar;               // [R P,H,U]
};

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
// then pg_reduce as after the pathwise sweep.  Box terms enter G, so they enter the gradient.
struct PsDev : PtPolicy {
    long long T;                                        // R P rows
    const double* eps; const double* traj; const double* step_reward; const double* step_risk;
    const double* var;                                  // [H,T,Ds] the forward's predicted variances
    double* G;                                          // [H-1,T] return-to-go
    double* S;                                          // [R,H] per-(restart, step) sums of G
    double* gmean; double* gvar;                        // [H-1,T,Ds] the VJP's cotangents
    const double* gxt;                                  // [H-1,T,D] the VJP's outputs
    double* zbar;                                       // [T,H,U]
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
    if (t == H - 1) {                                   // x_H carries no reward
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

// ---- host side ------------------------------------------------------------------------------------------------------
// Offsets in doubles into a particle workspace, for all four layouts (a slot a layout does not have stays 0); the
// predict (pws) and VJP (vws) workspaces are one slot when one call needs both.  total in bytes; 0 for unsupported
// sizes and on size_t overflow.
struct PtWs {
    size_t xt, mean, var;                               // forward: x~ [H or 1,T,D], step closure mean [T,Ds], var
    size_t mu, s2, W, Kh, L;                            // consistent forward: predict outputs, W_t, K* history, factor
    size_t gx, gvar, gxt, zbar, s1, s2r, gbeta, gy;     // reverse sweep and the policy-parameter reduction
    size_t G, dir;                                      // reverse of the conditioning (score: G = the return-to-go)
    size_t gsum;                                        // score: the per-(restart, step) sums of G
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

// the marginal rollout: x~, the predict outputs and one predict workspace at T = P
static PtWs pt_ws_layout(const pilco_particles* pr) {
    const size_t P = pr->P, Ds = pr->pol.Ds, D = pr->dyn.D;
    PtWs L = {}; PtTake take;
    L.xt = take({P, D}); L.mean = take({P, Ds}); L.var = take({P, Ds});
    L.pws_bytes = pilco_gp_predict_workspace_bytes(pr->dyn.n, pr->dyn.D, (int)Ds, pr->P, 0);
    L.pws = take({L.pws_bytes / sizeof(double)});
    L.total = L.pws_bytes ? take.bytes() : 0;
    return L;
}

// the gradient for R restarts: the forward's predict inputs and variances of EVERY step (the reverse sweep needs
// them), the state cotangent, the VJP's cotangents and output, z_bar of every point, the RBF sums, and one predict /
// VJP workspace at T = R P (never in use at the same time).  Rows are restart-major (row r P + p); nothing of size
// [., n] is kept.
static PtWs pg_ws_layout(const pilco_particles* pr, int R) {
    const size_t T = (size_t)R * pr->P, H = pr->H, Ds = pr->pol.Ds, U = pr->pol.U, D = pr->dyn.D;
    const size_t bf = pt_rbf(pr) ? pr->pol.rbf.n : 0;
    PtWs L = {}; PtTake take;
    L.xt = take({H, T, D}); L.mean = take({T, Ds}); L.var = take({H, T, Ds});
    L.gx = take({T, Ds}); L.gvar = take({T, Ds}); L.gxt = take({T, D}); L.zbar = take({T, H, U});
    L.s1 = take({(size_t)R, U, bf, Ds}); L.s2r = take({(size_t)R, U, bf, Ds});
    L.gbeta = take({(size_t)R, U, bf}); L.gy = take({(size_t)R, U, bf});
    const size_t pb = pilco_gp_predict_workspace_bytes(pr->dyn.n, pr->dyn.D, (int)Ds, (int)T, 0);
    const size_t vb = pilco_gp_predict_vjp_workspace_bytes(pr->dyn.n, pr->dyn.D, pr->dyn.E, (int)T);
    L.pws_bytes = L.vws_bytes = (pb && vb) ? (pb > vb ? pb : vb) : 0;
    L.pws = L.vws = take({L.pws_bytes / sizeof(double)});
    L.total = L.pws_bytes ? take.bytes() : 0;
    return L;
}

// the consistent rollout at T rows: x~ of every step [H,T,D], the predict outputs mu and var and the step closure's
// mean and var [T,Ds], W_t [E,T,np], the K* history [H,E,T,np], the packed factor rows [H(H+1)/2,E,T], one predict
// workspace at T
static void fs_take(const pilco_particles* pr, size_t T, PtWs& L, PtTake& take) {
    const size_t H = pr->H, Ds = pr->pol.Ds, D = pr->dyn.D, np = (size_t)pad64(pr->dyn.n);
    L.xt = take({H, T, D}); L.mu = take({T, Ds}); L.s2 = take({T, Ds}); L.mean = take({T, Ds}); L.var = take({T, Ds});
    L.W = take({T, Ds, np}); L.Kh = take({H, T, Ds, np}); L.L = take({H * (H + 1) / 2, T, Ds});
    L.pws_bytes = pilco_gp_predict_workspace_bytes(pr->dyn.n, pr->dyn.D, (int)Ds, (int)T, 0);
    L.pws = take({L.pws_bytes / sizeof(double)});
}

static PtWs fs_ws_layout(const pilco_particles* pr) {
    PtWs L = {}; PtTake take;
    fs_take(pr, pr->P, L, take);
    L.total = L.pws_bytes ? take.bytes() : 0;
    return L;
}

// the consistent gradient for R restarts: the consistent forward's at T = R P (its W slot holds a_t in the reverse
// sweep), then the var' history [H,T,Ds] (in place of the forward's single var slot), the packed cotangent rows
// [H(H+1)/2,E,T], the direct sums [E,T,D], x_bar and var_bar [T,Ds], the VJP output [T,D], z_bar [T,H,U], the RBF
// sums [R,U,bf,Ds] x 2 and [R,U,bf] x 2, and one VJP workspace at T
static PtWs fg_ws_layout(const pilco_particles* pr, int R) {
    const size_t T = (size_t)R * pr->P, H = pr->H, Ds = pr->pol.Ds, U = pr->pol.U, D = pr->dyn.D;
    const size_t bf = pt_rbf(pr) ? pr->pol.rbf.n : 0;
    PtWs L = {}; PtTake take;
    fs_take(pr, T, L, take);                            // pt_batch_ok: R P <= PT_MAX_P
    L.var = take({H, T, Ds}); L.G = take({H * (H + 1) / 2, T, Ds}); L.dir = take({T, Ds, D});
    L.gx = take({T, Ds}); L.gvar = take({T, Ds}); L.gxt = take({T, D}); L.zbar = take({T, H, U});
    L.s1 = take({(size_t)R, U, bf, Ds}); L.s2r = take({(size_t)R, U, bf, Ds});
    L.gbeta = take({(size_t)R, U, bf}); L.gy = take({(size_t)R, U, bf});
    L.vws_bytes = pilco_gp_predict_vjp_workspace_bytes(pr->dyn.n, pr->dyn.D, pr->dyn.E, (int)T);
    L.vws = take({L.vws_bytes / sizeof(double)});
    L.total = L.pws_bytes && L.vws_bytes ? take.bytes() : 0;
    return L;
}

// steps per pilco_gp_predict_vjp call of the score gradient: whole steps of T rows, at most PT_MAX_P rows (T <= PT_MAX_P)
static int ps_group(long long T, int H) {
    const long long k = PT_MAX_P / T;
    return H - 1 < k ? H - 1 : (int)k;
}

// the score gradient for R restarts: pg_ws_layout's forward part (x~ [H,T,D], mean [T,Ds], var [H,T,Ds]), then G
// [H-1,T], the sums [R,H], gmean and gvar [H-1,T,Ds], the VJP output [H-1,T,D], z_bar [T,H,U], the RBF sums
// [R,U,bf,Ds] x 2 and [R,U,bf] x 2, and one predict / VJP workspace for the predict at T and the largest VJP group.
// 0 also where the per-(step, particle) grids would pass 2^31 - 1 CTAs.
static PtWs ps_ws_layout(const pilco_particles* pr, int R) {
    const size_t T = (size_t)R * pr->P, H = pr->H, Hm = H > 0 ? H - 1 : 0, Ds = pr->pol.Ds, U = pr->pol.U;
    const size_t D = pr->dyn.D, bf = pt_rbf(pr) ? pr->pol.rbf.n : 0;
    PtWs L = {}; PtTake take;
    L.xt = take({H, T, D}); L.mean = take({T, Ds}); L.var = take({H, T, Ds});
    L.G = take({Hm, T}); L.gsum = take({(size_t)R, H});
    L.gx = take({Hm, T, Ds}); L.gvar = take({Hm, T, Ds}); L.gxt = take({Hm, T, D}); L.zbar = take({T, H, U});
    L.s1 = take({(size_t)R, U, bf, Ds}); L.s2r = take({(size_t)R, U, bf, Ds});
    L.gbeta = take({(size_t)R, U, bf}); L.gy = take({(size_t)R, U, bf});
    const int grp = ps_group((long long)T, (int)H);
    const size_t pb = pilco_gp_predict_workspace_bytes(pr->dyn.n, pr->dyn.D, (int)Ds, (int)T, 0);
    const size_t vb = pilco_gp_predict_vjp_workspace_bytes(pr->dyn.n, pr->dyn.D, pr->dyn.E, (int)T * (grp > 1 ? grp : 1));
    L.pws_bytes = L.vws_bytes = (pb && vb) ? (pb > vb ? pb : vb) : 0;
    L.pws = L.vws = take({L.pws_bytes / sizeof(double)});
    const size_t nb = (pr->P + PT_THREADS - 1) / PT_THREADS;
    L.total = L.pws_bytes && nb * H <= 0x7fffffff ? take.bytes() : 0;
    return L;
}

static bool pt_sizes_ok(const pilco_particles* pr) {
    return pr->P >= 1 && pr->P <= PT_MAX_P && pr->H >= 0 && pr->dyn.n >= 1 && pr->dyn.D >= 1 && pr->dyn.D <= MAXD &&
           pr->pol.Ds >= 1 && pr->pol.U >= 1 && pr->pol.Ds <= MAXE;
}

// R restarts of P particles: one CTA row per restart (gridDim.y) and R P predict points
static bool pt_batch_ok(int P, int R) {
    return R >= 1 && R <= 65535 && (long long)R * P <= PT_MAX_P;
}

// everything but the workspace (the gradients bring their own).  batched: the policy's batch strides are honoured
// (the batch_grad and consistent_grad entry points); otherwise a batched policy is unsupported.
static int pt_check_desc(const pilco_particles* pr, bool batched = false) {
    if (!pr) return PILCO_ERR_NULL;
    if (pr->P < 1 || pr->P > PT_MAX_P || pr->H < 0) return PILCO_ERR_DIM;
    const pilco_gp_model& g = pr->dyn;
    if (!g.X || !g.ell || !g.sf2 || !g.beta) return PILCO_ERR_NULL;
    if (g.mode != 0 || !g.iK || g.X_bs || g.ell_bs || g.sf2_bs || g.beta_bs) return PILCO_ERR_UNSUPPORTED;
    if (g.n < 1 || g.D < 1 || g.D > MAXD || g.E < 1 || g.E > MAXE || g.ldk < pad64(g.n)) return PILCO_ERR_DIM;
    const pilco_policy& pol = pr->pol;
    const int Ds = pol.Ds, U = pol.U;
    if (Ds < 1 || U < 1 || Ds + U != g.D || g.E != Ds) return PILCO_ERR_DIM;
    auto strides = [batched](std::initializer_list<long long> bs) {
        for (long long b : bs) {
            if (b && !batched) return PILCO_ERR_UNSUPPORTED;
            if (b < 0) return PILCO_ERR_DIM;
        }
        return PILCO_OK;
    };
    if (pol.kind == PILCO_POLICY_LINEAR) {
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
    if (pr->n_rewards < 1 || pr->n_rewards > 8) return PILCO_ERR_DIM;
    for (int k = 0; k < pr->n_rewards; ++k) {
        const pilco_reward_term& rt = pr->rewards[k];
        if (!rt.W) return PILCO_ERR_NULL;
        if (rt.kind != PILCO_REWARD_EXP && rt.kind != PILCO_REWARD_LINEAR && rt.kind != PILCO_REWARD_BOX) return PILCO_ERR_UNSUPPORTED;
        if (rt.channel != PILCO_CHANNEL_ADD && rt.channel != PILCO_CHANNEL_MULT) return PILCO_ERR_UNSUPPORTED;
        if (rt.kind == PILCO_REWARD_EXP && !rt.t) return PILCO_ERR_NULL;
    }
    if (!pr->x0 || !pr->eps || !pr->traj || !pr->act || !pr->step_reward || !pr->step_risk || !pr->ret)
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

// the gradient's output pointers, after pt_check_desc
static int pg_check(const pilco_particles* pr, const pilco_particles_grad* g) {
    if (!g || !g->value || !g->ws) return PILCO_ERR_NULL;
    if (pt_rbf(pr) ? (!g->gXc || !g->gYc || !g->gell || !g->pol_L) : (!g->gW || !g->gb)) return PILCO_ERR_NULL;
    return PILCO_OK;
}

static PtPolicy pt_policy(const pilco_particles* pr) {
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
    a.n_rewards = pr->n_rewards; a.n_mult = 0;
    for (int k = 0; k < 8; ++k) a.rewards[k] = pr->rewards[k];
    for (int k = 0; k < pr->n_rewards; ++k) a.n_mult += pr->rewards[k].channel == PILCO_CHANNEL_MULT;
    a.mult_mu = pr->mult_mu;
    return a;
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
// kept when either needs it.
static int pt_forward(const pilco_particles* pr, int R, double* ws, const PtWs& L, bool consistent, bool history,
                      cudaStream_t st) {
    const int P = pr->P, H = pr->H, Ds = pr->pol.Ds, D = pr->dyn.D, T = R * P, np = pad64(pr->dyn.n);
    const size_t TD = (size_t)T * D, TDs = (size_t)T * Ds, slot = TDs * np;
    const size_t xstep = consistent || history ? TD : 0, vstep = history ? TDs : 0;
    const dim3 grid((P + PT_THREADS - 1) / PT_THREADS, R), cgrid((P + FS_WARPS - 1) / FS_WARPS, Ds, R);
    PtDev a;
    static_cast<PtPolicy&>(a) = pt_policy(pr);
    a.x0 = pr->x0; a.eps = pr->eps;
    a.traj = pr->traj; a.act = pr->act; a.step_reward = pr->step_reward; a.step_risk = pr->step_risk; a.ret = pr->ret;
    a.mean = ws + L.mean;
    FsCond c;
    c.P = P; c.T = T; c.H = H; c.D = D; c.Ds = Ds; c.n = pr->dyn.n; c.np = np; c.t = 0;
    c.ell = pr->dyn.ell; c.sf2 = pr->dyn.sf2;
    c.xh = ws + L.xt; c.mu = ws + L.mu; c.s2 = ws + L.s2; c.W = ws + L.W; c.Kh = ws + L.Kh;
    c.eps = pr->eps; c.L = ws + L.L; c.mean = ws + L.mean;
    for (int t = 0; t <= H; ++t) {
        a.t = t;
        a.xt = ws + L.xt + (size_t)(t < H ? t : 0) * xstep;
        a.var = ws + L.var + (size_t)(t > 0 ? t - 1 : 0) * vstep;
        launch_hi(pt_step_kernel, grid, dim3(PT_THREADS), 0, st, a);
        CUDA_LAUNCH_CHECK();
        if (t == H) break;
        double* var = ws + L.var + (size_t)t * vstep;
        if (consistent) {
            const int rc = fs_predict_launch(st, &pr->dyn, T, a.xt, ws + L.mu, ws + L.s2, ws + L.W, ws + L.Kh + t * slot,
                                             ws + L.pws);
            if (rc) return rc;
            c.t = t; c.var = var;
            launch_hi(fs_cond_kernel, cgrid, dim3(FS_WARPS * 32), 0, st, c);
            CUDA_LAUNCH_CHECK();
        } else {
            const int rc = pilco_gp_predict(&pr->dyn, 0, Ds, T, a.xt, ws + L.mean, var, 0, ws + L.pws, L.pws_bytes, st);
            if (rc) return rc;
        }
    }
    return PILCO_OK;
}

void chol_solve_vec_launch(cudaStream_t st, int batch, int n, const double* L, int ld, long long ms, int E,
                           const double* Y, long long Y_bs, long long y_es, int yinc, double* x, long long xs);
int rbf_factor_bwd_launch(cudaStream_t st, int R, int bf, int Ds, int U, const double* X, long long X_bs,
                          const double* ell, long long ell_bs, const double* sf2, long long sf2_bs,
                          const double* beta, long long beta_bs, const double* gy,
                          double* gX, double* gY, double* gell);

// value and the policy-parameter gradient over all P H points of each restart, fixed order, from z_bar [R P,H,U]
static int pg_reduce(const pilco_particles* pr, int R, const pilco_particles_grad* g, double* ws, const PtWs& L,
                     cudaStream_t st) {
    PgRed r;
    static_cast<PtPolicy&>(r) = pt_policy(pr);
    const bool rbf = r.pol_kind == PILCO_POLICY_RBF;
    const int Ds = r.Ds, U = r.U, bf = r.bf;
    r.traj = pr->traj; r.zbar = ws + L.zbar; r.ret = pr->ret;
    r.gW = g->gW; r.gb = g->gb;
    r.s1 = ws + L.s1; r.s2 = ws + L.s2r; r.gbeta = ws + L.gbeta;
    r.gXc = g->gXc; r.gell = g->gell;
    r.value = g->value;
    launch_hi(pg_param_kernel, dim3((rbf ? U * bf : U) + 1, R), dim3(256), 0, st, r);
    CUDA_LAUNCH_CHECK();
    if (rbf) {                                          // through beta = (K + sn2 I)^-1 Yc, as pilco_rollout_backward
        const int ldw = pad64(bf);
        launch_hi(pg_rbf_finish_kernel, dim3(R), dim3(128), 0, st, r);
        CUDA_LAUNCH_CHECK();
        chol_solve_vec_launch(st, R * U, bf, g->pol_L, ldw, (long long)ldw * ldw, U,
                              r.gbeta, (long long)U * bf, bf, 1, ws + L.gy, bf);
        const int rc = rbf_factor_bwd_launch(st, R, bf, Ds, U, r.C, r.C_bs, r.ell, r.ell_bs, r.sf2, r.sf2_bs,
                                             r.beta, r.beta_bs, ws + L.gy, g->gXc, g->gYc, g->gell);
        if (rc) return rc;
    }
    return PILCO_OK;
}

// The reverse sweep after pt_forward(history) and the reduction (DESIGN.md sections 12, 15):
//   pg_step<H-1>, [VJP<t>, pg_step<t>] for t = H-2 .. 0, then pg_reduce's launches
// The step's VJP is pilco_gp_predict_vjp, or (consistent) fs_cond_bwd_kernel followed by fs_predict_vjp_kernel.
static int pg_reverse(const pilco_particles* pr, int R, const pilco_particles_grad* g, const PtWs& L, bool consistent,
                      cudaStream_t st) {
    double* ws = (double*)g->ws;
    const int P = pr->P, H = pr->H, Ds = pr->pol.Ds, D = pr->dyn.D, T = R * P;
    const size_t TD = (size_t)T * D, TDs = (size_t)T * Ds;
    const dim3 grid((P + PT_THREADS - 1) / PT_THREADS, R), cgrid((P + FS_WARPS - 1) / FS_WARPS, Ds, R);
    if (consistent && H > 1) cudaMemsetAsync(ws + L.G, 0, (size_t)H * (H + 1) / 2 * TDs * sizeof(double), st);
    PgDev b;
    static_cast<PtPolicy&>(b) = pt_policy(pr);
    b.eps = pr->eps; b.traj = pr->traj; b.step_risk = pr->step_risk;
    b.gx = ws + L.gx; b.gvar = ws + L.gvar; b.zbar = ws + L.zbar;
    FsBwd q;                                            // the cotangent rows G accumulate from zero
    q.P = P; q.T = T; q.H = H; q.D = D; q.Ds = Ds; q.np = pad64(pr->dyn.n); q.t = 0;
    q.ell = pr->dyn.ell; q.sf2 = pr->dyn.sf2;
    q.xh = ws + L.xt; q.Kh = ws + L.Kh; q.L = ws + L.L; q.eps = pr->eps;
    q.gx = b.gx; q.gvar = b.gvar; q.G = ws + L.G; q.A = ws + L.W; q.dir = ws + L.dir;
    for (int t = H - 1; t >= 0; --t) {
        b.t = t;
        b.gxt = nullptr;
        if (t < H - 1) {
            const double* xt = ws + L.xt + (size_t)t * TD;
            int rc;
            if (consistent) {
                q.t = t;
                launch_hi(fs_cond_bwd_kernel, cgrid, dim3(FS_WARPS * 32), 0, st, q);
                CUDA_LAUNCH_CHECK();
                rc = fs_vjp_launch(st, &pr->dyn, T, xt, b.gx, q.A, q.dir, ws + L.gxt, ws + L.vws);
            } else {
                rc = pilco_gp_predict_vjp(&pr->dyn, T, xt, b.gx, b.gvar, ws + L.gxt, ws + L.vws, L.vws_bytes, st);
            }
            if (rc) return rc;
            b.gxt = ws + L.gxt;
        }
        b.var_prev = t > 0 ? ws + L.var + (size_t)(t - 1) * TDs : nullptr;
        launch_hi(pg_step_kernel, grid, dim3(PT_THREADS), 0, st, b);
        CUDA_LAUNCH_CHECK();
    }
    return pg_reduce(pr, R, g, ws, L, st);
}

// the validated gradient of R restarts: the forward with its history, then the reverse sweep
static int pg_run(const pilco_particles* pr, int R, const pilco_particles_grad* g, bool consistent,
                  pilco_stream_t stream) {
    const PtWs L = consistent ? fg_ws_layout(pr, R) : pg_ws_layout(pr, R);
    if (const int rc = pt_check_ws(g->ws, g->ws_bytes, L.total)) return rc;
    if (consistent) {
        if (const int rc = fs_predict_prepare()) return rc;
        if (const int rc = fs_vjp_prepare()) return rc;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (const int rc = pt_forward(pr, R, (double*)g->ws, L, consistent, true, st)) return rc;
    return pg_reverse(pr, R, g, L, consistent, st);
}

// the forward alone, R = 1
static int pt_run(const pilco_particles* pr, bool consistent, pilco_stream_t stream) {
    if (const int rc = pt_check_desc(pr)) return rc;
    const PtWs L = consistent ? fs_ws_layout(pr) : pt_ws_layout(pr);
    if (const int rc = pt_check_ws(pr->ws, pr->ws_bytes, L.total)) return rc;
    if (consistent)
        if (const int rc = fs_predict_prepare()) return rc;
    return pt_forward(pr, 1, (double*)pr->ws, L, consistent, false, (cudaStream_t)stream);
}

// The score-function gradient of R restarts (validated; DESIGN.md section 16):
//   pt_forward(history), ps_togo, ps_base, ps_cot, VJP of steps 0..H-2 in groups of whole steps, ps_zbar, pg_reduce
// The x~ history [H-1,T,D] and the cotangents [H-1,T,Ds] are contiguous, so a group of k steps is one VJP call at k T
// rows; a point's VJP does not depend on T or on its row, so the grouping changes no bit.
static int ps_run(const pilco_particles* pr, int R, const pilco_particles_grad* g, pilco_stream_t stream) {
    const PtWs L = ps_ws_layout(pr, R);
    if (const int rc = pt_check_ws(g->ws, g->ws_bytes, L.total)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    double* ws = (double*)g->ws;
    if (const int rc = pt_forward(pr, R, ws, L, false, true, st)) return rc;
    const int P = pr->P, H = pr->H, Ds = pr->pol.Ds, D = pr->dyn.D, T = R * P, nb = (P + PT_THREADS - 1) / PT_THREADS;
    PsDev a;
    static_cast<PtPolicy&>(a) = pt_policy(pr);
    a.T = T;
    a.eps = pr->eps; a.traj = pr->traj; a.step_reward = pr->step_reward; a.step_risk = pr->step_risk;
    a.var = ws + L.var; a.G = ws + L.G; a.S = ws + L.gsum; a.gmean = ws + L.gx; a.gvar = ws + L.gvar;
    a.gxt = ws + L.gxt; a.zbar = ws + L.zbar;
    if (H > 1) {
        launch_hi(ps_togo_kernel, dim3(nb, R), dim3(PT_THREADS), 0, st, a);
        CUDA_LAUNCH_CHECK();
        launch_hi(ps_base_kernel, dim3(H - 1, R), dim3(256), 0, st, a);
        CUDA_LAUNCH_CHECK();
        launch_hi(ps_cot_kernel, dim3(nb * (H - 1), R), dim3(PT_THREADS), 0, st, a);
        CUDA_LAUNCH_CHECK();
        const int grp = ps_group(T, H);
        for (int t0 = 0; t0 < H - 1; t0 += grp) {
            const int k = grp < H - 1 - t0 ? grp : H - 1 - t0;
            const size_t o = (size_t)t0 * T;
            const int rc = pilco_gp_predict_vjp(&pr->dyn, k * T, ws + L.xt + o * D, ws + L.gx + o * Ds,
                                                ws + L.gvar + o * Ds, ws + L.gxt + o * D, ws + L.vws, L.vws_bytes, st);
            if (rc) return rc;
        }
    }
    if (H > 0) {
        launch_hi(ps_zbar_kernel, dim3(nb * H, R), dim3(PT_THREADS), 0, st, a);
        CUDA_LAUNCH_CHECK();
    }
    return pg_reduce(pr, R, g, ws, L, st);
}

// everything a gradient entry point checks before its workspace: batched honours the policy's batch strides
static int pg_validate(const pilco_particles* pr, int R, const pilco_particles_grad* g, bool batched) {
    if (const int rc = pt_check_desc(pr, batched)) return rc;
    if (batched && !pt_batch_ok(pr->P, R)) return PILCO_ERR_DIM;
    return pg_check(pr, g);
}

static int pg_entry(const pilco_particles* pr, int R, const pilco_particles_grad* g, bool batched, bool consistent,
                    pilco_stream_t stream) {
    if (const int rc = pg_validate(pr, R, g, batched)) return rc;
    return pg_run(pr, R, g, consistent, stream);
}

extern "C" {

size_t pilco_particles_workspace_bytes(const pilco_particles* pr) {
    return pr && pt_sizes_ok(pr) ? pt_ws_layout(pr).total : 0;
}

int pilco_particles_rollout(const pilco_particles* pr, pilco_stream_t stream) {
    return pt_run(pr, false, stream);
}

size_t pilco_particles_grad_workspace_bytes(const pilco_particles* pr) {
    return pr && pt_sizes_ok(pr) ? pg_ws_layout(pr, 1).total : 0;
}

int pilco_particles_rollout_grad(const pilco_particles* pr, const pilco_particles_grad* g, pilco_stream_t stream) {
    return pg_entry(pr, 1, g, false, false, stream);
}

size_t pilco_particles_batch_grad_workspace_bytes(const pilco_particles* pr, int R) {
    return pr && pt_sizes_ok(pr) && pt_batch_ok(pr->P, R) ? pg_ws_layout(pr, R).total : 0;
}

int pilco_particles_rollout_batch_grad(const pilco_particles* pr, int R, const pilco_particles_grad* g,
                                       pilco_stream_t stream) {
    return pg_entry(pr, R, g, true, false, stream);
}

size_t pilco_particles_consistent_workspace_bytes(const pilco_particles* pr) {
    return pr && pt_sizes_ok(pr) ? fs_ws_layout(pr).total : 0;
}

int pilco_particles_rollout_consistent(const pilco_particles* pr, pilco_stream_t stream) {
    return pt_run(pr, true, stream);
}

size_t pilco_particles_consistent_grad_workspace_bytes(const pilco_particles* pr, int R) {
    return pr && pt_sizes_ok(pr) && pt_batch_ok(pr->P, R) ? fg_ws_layout(pr, R).total : 0;
}

int pilco_particles_rollout_consistent_grad(const pilco_particles* pr, int R, const pilco_particles_grad* g,
                                            pilco_stream_t stream) {
    return pg_entry(pr, R, g, true, true, stream);
}

size_t pilco_particles_score_grad_workspace_bytes(const pilco_particles* pr, int R) {
    return pr && pt_sizes_ok(pr) && pt_batch_ok(pr->P, R) ? ps_ws_layout(pr, R).total : 0;
}

int pilco_particles_rollout_score_grad(const pilco_particles* pr, int R, const pilco_particles_grad* g,
                                       pilco_stream_t stream) {
    if (const int rc = pg_validate(pr, R, g, true)) return rc;
    return ps_run(pr, R, g, stream);
}

}  // extern "C"
