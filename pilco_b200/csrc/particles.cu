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
#include <initializer_list>
#include "common.cuh"
#include "risk_math.cuh"

#define PT_THREADS 128
#define PT_MAX_P   (65535 * 32)         // pilco_gp_predict's T limit
#define PT_RBF_VAR 1e-6                 // output variance of the deterministic-GP policy (mode 1, mm_finish_device)
#define PT_INV_PI  0.31830988618379067154

struct PtDev {
    int P, H, Ds, U, t;
    int pol_kind, squash;
    const double* maxa;
    const double* W; const double* b;                   // linear policy [U,Ds], [U]
    const double* C; const double* ell; const double* sf2; const double* beta; int bf;   // RBF policy
    long long W_bs, b_bs, C_bs, ell_bs, sf2_bs, beta_bs;   // per-restart policy strides (0: shared)
    int n_rewards, n_mult; pilco_reward_term rewards[8]; double mult_mu;
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
struct PgDev {
    int P, H, Ds, U, t;
    int pol_kind, squash;
    const double* maxa;
    const double* W; const double* b;
    const double* C; const double* ell; const double* sf2; const double* beta; int bf;
    long long W_bs, b_bs, C_bs, ell_bs, sf2_bs, beta_bs;
    int n_rewards, n_mult; pilco_reward_term rewards[8]; double mult_mu;
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
    // policy: z_bar_t and (d pi / dx)' z_bar_t; z_t recomputed in the forward's order
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

struct PgRed {
    int P, H, Ds, U, bf, pol_kind;
    const double* traj; const double* zbar; const double* ret;
    const double* C; const double* ell; const double* sf2; const double* beta;
    long long C_bs, ell_bs, sf2_bs, beta_bs;            // per-restart RBF policy strides (0: shared)
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

struct FsCond {
    int P, H, D, Ds, n, np, t;
    const double* ell; const double* sf2;               // dynamics [E,D], [E]
    const double* xh;                                   // [H,P,D] predict inputs of the steps so far
    const double* mu; const double* s2;                 // [P,Ds] the posterior mean and variance at x~_t
    const double* W;                                    // [E,P,np] W_t = K*_t iK
    const double* Kh;                                   // [H,E,P,np] K*_s of every step
    const double* eps;                                  // [P,H,Ds]
    double* L;                                          // [H(H+1)/2, E, P] packed rows; (s, r) at s(s+1)/2 + r
    double* mean; double* var;                          // [P,Ds] what pt_step_kernel closes the step with
};

__device__ __forceinline__ double fs_bfly(double v) {   // fixed butterfly: every lane ends with the same bits
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// grid (ceil(P / FS_WARPS), E), one warp per (particle p, output e): step t's conditioning on the particle's past.
// The packed diagonal holds the pivot later substitutions divide by: sqrt(d2), or 0 for a degenerate column.
__global__ void __launch_bounds__(FS_WARPS * 32, 4) fs_cond_kernel(FsCond a) {
    PDL_ENTRY();
    const int lane = threadIdx.x & 31, p = blockIdx.x * FS_WARPS + (threadIdx.x >> 5), e = blockIdx.y;
    if (p >= a.P) return;
    const int D = a.D, Ds = a.Ds, t = a.t, n = a.n;
    const size_t P = a.P, EP = (size_t)Ds * P, pe = (size_t)e * P + p;
    const double sf2 = a.sf2[e];
    // lane d < D holds dimension d of x~_t and 1 / ell_ed
    const bool dl = lane < D;
    const double xd = dl ? a.xh[((size_t)t * P + p) * D + lane] : 0.0;
    const double ild = dl ? 1.0 / a.ell[(size_t)e * D + lane] : 0.0;
    double* Lt = a.L + (size_t)t * (t + 1) / 2 * EP + pe;              // row t: entry s at Lt[s EP]
    const double* __restrict__ Wr = a.W + pe * a.np;
    // c_s = k_e(x~_t, x~_s) - W_t . K*_s: lanes stride the columns (and the dimensions) in order, then the butterfly
    for (int s = 0; s < t; ++s) {
        const double* __restrict__ Kr = a.Kh + ((size_t)s * EP + pe) * a.np;
        double dot = 0.0;
#pragma unroll 4
        for (int j = lane; j < n; j += 32) dot = fma(Wr[j], Kr[j], dot);
        const double q = dl ? (xd - a.xh[((size_t)s * P + p) * D + lane]) * ild : 0.0;
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
        const size_t o = (size_t)p * Ds + e;
        const double mu = a.mu[o], d2 = a.s2[o] - ssq;
        Lt[(size_t)t * EP] = d2 > FS_TAU * sf2 ? sqrt(d2) : 0.0;
        a.mean[o] = t > 0 ? mu + sme : mu;              // t = 0: the marginal sampler's step exactly
        a.var[o] = d2 < 0.0 ? 0.0 : d2;                 // NaN stays NaN
    }
}

struct PtWs { size_t xt, mean, var, pws, pws_bytes, total; };     // offsets in doubles; total and pws_bytes in bytes

static PtWs pt_ws_layout(const pilco_particles* pr) {
    const size_t P = pr->P, Ds = pr->pol.Ds, D = pr->dyn.D;
    PtWs L; size_t o = 0;
    auto take = [&](size_t len) { const size_t at = o; o += (len + 1) & ~(size_t)1; return at; };
    L.xt = take(P * D); L.mean = take(P * Ds); L.var = take(P * Ds);
    L.pws = o;
    L.pws_bytes = pilco_gp_predict_workspace_bytes(pr->dyn.n, pr->dyn.D, (int)Ds, pr->P, 0);
    L.total = o * sizeof(double) + L.pws_bytes;
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

// everything but the workspace (pilco_particles_rollout_grad brings its own).  batched: the policy's batch strides
// are honoured (pilco_particles_rollout_batch_grad); otherwise a batched policy is unsupported.
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

static int pt_check(const pilco_particles* pr) {
    const int rc = pt_check_desc(pr);
    if (rc) return rc;
    if (!pr->ws) return PILCO_ERR_NULL;
    if ((uintptr_t)pr->ws & 15) return PILCO_ERR_ALIGN;
    const PtWs L = pt_ws_layout(pr);
    if (L.pws_bytes == 0) return PILCO_ERR_DIM;
    if (pr->ws_bytes < L.total) return PILCO_ERR_WORKSPACE;
    return PILCO_OK;
}

static PtDev pt_dev(const pilco_particles* pr) {
    const pilco_policy& pol = pr->pol;
    PtDev a;
    a.P = pr->P; a.H = pr->H; a.Ds = pol.Ds; a.U = pol.U; a.t = 0;
    a.pol_kind = pol.kind; a.squash = pol.squash; a.maxa = pol.max_action;
    a.W = pol.W; a.b = pol.b;
    a.C = pol.rbf.X; a.ell = pol.rbf.ell; a.sf2 = pol.rbf.sf2; a.beta = pol.rbf.beta; a.bf = pol.rbf.n;
    const bool rbf = pol.kind == PILCO_POLICY_RBF;
    a.W_bs = rbf ? 0 : pol.W_bs; a.b_bs = rbf ? 0 : pol.b_bs;
    a.C_bs = rbf ? pol.rbf.X_bs : 0; a.ell_bs = rbf ? pol.rbf.ell_bs : 0;
    a.sf2_bs = rbf ? pol.rbf.sf2_bs : 0; a.beta_bs = rbf ? pol.rbf.beta_bs : 0;
    a.n_rewards = pr->n_rewards; a.n_mult = 0;
    for (int k = 0; k < 8; ++k) a.rewards[k] = pr->rewards[k];
    for (int k = 0; k < pr->n_rewards; ++k) a.n_mult += pr->rewards[k].channel == PILCO_CHANNEL_MULT;
    a.mult_mu = pr->mult_mu;
    a.x0 = pr->x0; a.eps = pr->eps;
    a.traj = pr->traj; a.act = pr->act; a.step_reward = pr->step_reward; a.step_risk = pr->step_risk; a.ret = pr->ret;
    return a;
}

// workspace of the consistent rollout (offsets in doubles; total and pws_bytes in bytes; ok = false on size_t
// overflow): x~ of every step [H,P,D], the predict outputs mu and var and the step closure's mean and var [P,Ds],
// W_t [E,P,np], the K* history [H,E,P,np], the packed factor rows [H(H+1)/2,E,P], one predict workspace at T = P
struct FsWs { size_t xh, mu, s2, mean, var, W, Kh, L, pws, pws_bytes, total; bool ok; };

static bool fs_mul(size_t x, size_t y, size_t& r) { return !__builtin_mul_overflow(x, y, &r); }

static FsWs fs_ws_layout(const pilco_particles* pr) {
    FsWs L = {};
    const size_t P = pr->P, H = pr->H, Ds = pr->pol.Ds, D = pr->dyn.D, np = (size_t)pad64(pr->dyn.n);
    size_t xh, pd, w, kh, rows, lp;
    L.ok = fs_mul(H * P, D, xh) && fs_mul(P, Ds, pd) && fs_mul(pd, np, w) && fs_mul(H, w, kh) &&
           fs_mul(H, H + 1, rows) && fs_mul(rows / 2, pd, lp);
    if (!L.ok) return L;
    size_t o = 0;
    auto take = [&](size_t len) {
        const size_t at = o;
        if (len == SIZE_MAX || __builtin_add_overflow(o, len + (len & 1), &o)) L.ok = false;
        return at;
    };
    L.xh = take(xh); L.mu = take(pd); L.s2 = take(pd); L.mean = take(pd); L.var = take(pd);
    L.W = take(w); L.Kh = take(kh); L.L = take(lp);
    L.pws = o;
    L.pws_bytes = pilco_gp_predict_workspace_bytes(pr->dyn.n, pr->dyn.D, (int)Ds, pr->P, 0);
    size_t b = 0;
    if (!L.ok || !fs_mul(o, sizeof(double), b) || __builtin_add_overflow(b, L.pws_bytes, &L.total)) L.ok = false;
    return L;
}

int fs_predict_prepare();
int fs_predict_launch(cudaStream_t st, const pilco_gp_model* gp, int T, const double* Xs, double* mean, double* var,
                      double* W, double* Ks, void* ws);

// workspace of the particle gradient for R restarts (offsets in doubles; total and pws_bytes in bytes): the forward's
// predict inputs and variances of EVERY step (the reverse sweep needs them), the state cotangent, the VJP's cotangents
// and output, z_bar of every point, the RBF sums, and one predict / VJP workspace at T = R P (never in use at the same
// time).  Rows are restart-major (row r P + p); nothing of size [., n] is kept.
struct PgWs { size_t xt, mean, var, gx, gvar, gxt, zbar, s1, s2, gbeta, gy, pws, pws_bytes, total; };

static PgWs pg_ws_layout(const pilco_particles* pr, int R) {
    const size_t T = (size_t)R * pr->P, H = pr->H, Ds = pr->pol.Ds, U = pr->pol.U, D = pr->dyn.D;
    const size_t bf = pr->pol.kind == PILCO_POLICY_RBF ? pr->pol.rbf.n : 0;
    PgWs L; size_t o = 0;
    auto take = [&](size_t len) { const size_t at = o; o += (len + 1) & ~(size_t)1; return at; };
    L.xt = take(H * T * D); L.mean = take(T * Ds); L.var = take(H * T * Ds);
    L.gx = take(T * Ds); L.gvar = take(T * Ds); L.gxt = take(T * D); L.zbar = take(T * H * U);
    L.s1 = take(R * U * bf * Ds); L.s2 = take(R * U * bf * Ds); L.gbeta = take(R * U * bf); L.gy = take(R * U * bf);
    L.pws = o;
    const size_t pb = pilco_gp_predict_workspace_bytes(pr->dyn.n, pr->dyn.D, (int)Ds, (int)T, 0);
    const size_t vb = pilco_gp_predict_vjp_workspace_bytes(pr->dyn.n, pr->dyn.D, pr->dyn.E, (int)T);
    L.pws_bytes = (pb && vb) ? (pb > vb ? pb : vb) : 0;
    L.total = o * sizeof(double) + L.pws_bytes;
    return L;
}

void chol_solve_vec_launch(cudaStream_t st, int batch, int n, const double* L, int ld, long long ms, int E,
                           const double* Y, long long Y_bs, long long y_es, int yinc, double* x, long long xs);
int rbf_factor_bwd_launch(cudaStream_t st, int R, int bf, int Ds, int U, const double* X, long long X_bs,
                          const double* ell, long long ell_bs, const double* sf2, long long sf2_bs,
                          const double* beta, long long beta_bs, const double* gy,
                          double* gX, double* gY, double* gell);

// the gradient's arguments and workspace, after pt_check_desc
static int pg_check(const pilco_particles* pr, int R, const pilco_particles_grad* g) {
    if (!g || !g->value || !g->ws) return PILCO_ERR_NULL;
    const bool rbf = pr->pol.kind == PILCO_POLICY_RBF;
    if (rbf ? (!g->gXc || !g->gYc || !g->gell || !g->pol_L) : (!g->gW || !g->gb)) return PILCO_ERR_NULL;
    if ((uintptr_t)g->ws & 15) return PILCO_ERR_ALIGN;
    const PgWs L = pg_ws_layout(pr, R);
    if (L.pws_bytes == 0) return PILCO_ERR_DIM;
    if (g->ws_bytes < L.total) return PILCO_ERR_WORKSPACE;
    return PILCO_OK;
}

// forward rollout and reverse sweep of R restarts (validated): R = 1 is pilco_particles_rollout_grad
static int pg_run(const pilco_particles* pr, int R, const pilco_particles_grad* g, pilco_stream_t stream) {
    const PgWs L = pg_ws_layout(pr, R);
    cudaStream_t st = (cudaStream_t)stream;
    double* ws = (double*)g->ws;
    const pilco_policy& pol = pr->pol;
    const bool rbf = pol.kind == PILCO_POLICY_RBF;
    const int P = pr->P, H = pr->H, Ds = pol.Ds, U = pol.U, D = Ds + U, T = R * P;
    const size_t PD = (size_t)T * D, PDs = (size_t)T * Ds;
    const dim3 grid((P + PT_THREADS - 1) / PT_THREADS, R);
    int rc;
    // forward: pilco_particles_rollout's launches, with the predict inputs and variances of every step kept
    PtDev a = pt_dev(pr);
    a.mean = ws + L.mean;
    for (int t = 0; t <= H; ++t) {
        a.t = t;
        a.xt = ws + L.xt + (size_t)(t < H ? t : 0) * PD;
        a.var = ws + L.var + (size_t)(t > 0 ? t - 1 : 0) * PDs;
        launch_hi(pt_step_kernel, grid, dim3(PT_THREADS), 0, st, a);
        CUDA_LAUNCH_CHECK();
        if (t == H) break;
        rc = pilco_gp_predict(&pr->dyn, 0, Ds, T, a.xt, ws + L.mean, ws + L.var + (size_t)t * PDs, 0,
                              ws + L.pws, L.pws_bytes, stream);
        if (rc) return rc;
    }
    // reverse sweep
    PgDev b;
    b.P = P; b.H = H; b.Ds = Ds; b.U = U;
    b.pol_kind = pol.kind; b.squash = pol.squash; b.maxa = pol.max_action;
    b.W = pol.W; b.b = pol.b;
    b.C = pol.rbf.X; b.ell = pol.rbf.ell; b.sf2 = pol.rbf.sf2; b.beta = pol.rbf.beta; b.bf = pol.rbf.n;
    b.W_bs = a.W_bs; b.b_bs = a.b_bs; b.C_bs = a.C_bs; b.ell_bs = a.ell_bs; b.sf2_bs = a.sf2_bs; b.beta_bs = a.beta_bs;
    b.n_rewards = a.n_rewards; b.n_mult = a.n_mult; b.mult_mu = a.mult_mu;
    for (int k = 0; k < 8; ++k) b.rewards[k] = a.rewards[k];
    b.eps = pr->eps; b.traj = pr->traj; b.step_risk = pr->step_risk;
    b.gx = ws + L.gx; b.gvar = ws + L.gvar; b.zbar = ws + L.zbar;
    for (int t = H - 1; t >= 0; --t) {
        b.t = t;
        b.gxt = nullptr;
        if (t < H - 1) {
            rc = pilco_gp_predict_vjp(&pr->dyn, T, ws + L.xt + (size_t)t * PD, b.gx, b.gvar, ws + L.gxt,
                                      ws + L.pws, L.pws_bytes, stream);
            if (rc) return rc;
            b.gxt = ws + L.gxt;
        }
        b.var_prev = t > 0 ? ws + L.var + (size_t)(t - 1) * PDs : nullptr;
        launch_hi(pg_step_kernel, grid, dim3(PT_THREADS), 0, st, b);
        CUDA_LAUNCH_CHECK();
    }
    // value and the policy-parameter gradient over all P H points of each restart, fixed order
    PgRed r;
    r.P = P; r.H = H; r.Ds = Ds; r.U = U; r.bf = rbf ? pol.rbf.n : 0; r.pol_kind = pol.kind;
    r.traj = pr->traj; r.zbar = ws + L.zbar; r.ret = pr->ret;
    r.C = pol.rbf.X; r.ell = pol.rbf.ell; r.sf2 = pol.rbf.sf2; r.beta = pol.rbf.beta;
    r.C_bs = a.C_bs; r.ell_bs = a.ell_bs; r.sf2_bs = a.sf2_bs; r.beta_bs = a.beta_bs;
    r.gW = g->gW; r.gb = g->gb;
    r.s1 = ws + L.s1; r.s2 = ws + L.s2; r.gbeta = ws + L.gbeta;
    r.gXc = g->gXc; r.gell = g->gell;
    r.value = g->value;
    launch_hi(pg_param_kernel, dim3((rbf ? U * r.bf : U) + 1, R), dim3(256), 0, st, r);
    CUDA_LAUNCH_CHECK();
    if (rbf) {                                          // through beta = (K + sn2 I)^-1 Yc, as pilco_rollout_backward
        const int bf = r.bf, ldw = pad64(bf);
        launch_hi(pg_rbf_finish_kernel, dim3(R), dim3(128), 0, st, r);
        CUDA_LAUNCH_CHECK();
        chol_solve_vec_launch(st, R * U, bf, g->pol_L, ldw, (long long)ldw * ldw, U,
                              ws + L.gbeta, (long long)U * bf, bf, 1, ws + L.gy, bf);
        rc = rbf_factor_bwd_launch(st, R, bf, Ds, U, pol.rbf.X, a.C_bs, pol.rbf.ell, a.ell_bs, pol.rbf.sf2, a.sf2_bs,
                                   pol.rbf.beta, a.beta_bs, ws + L.gy, g->gXc, g->gYc, g->gell);
        if (rc) return rc;
    }
    return PILCO_OK;
}

extern "C" {

size_t pilco_particles_workspace_bytes(const pilco_particles* pr) {
    if (!pr || !pt_sizes_ok(pr)) return 0;
    const PtWs L = pt_ws_layout(pr);
    return L.pws_bytes ? L.total : 0;
}

int pilco_particles_rollout(const pilco_particles* pr, pilco_stream_t stream) {
    const int rc0 = pt_check(pr);
    if (rc0) return rc0;
    const PtWs L = pt_ws_layout(pr);
    cudaStream_t st = (cudaStream_t)stream;
    double* ws = (double*)pr->ws;
    const pilco_policy& pol = pr->pol;
    PtDev a = pt_dev(pr);
    a.xt = ws + L.xt; a.mean = ws + L.mean; a.var = ws + L.var;
    const dim3 grid((pr->P + PT_THREADS - 1) / PT_THREADS);
    for (int t = 0; t <= pr->H; ++t) {
        a.t = t;
        launch_hi(pt_step_kernel, grid, dim3(PT_THREADS), 0, st, a);
        CUDA_LAUNCH_CHECK();
        if (t == pr->H) break;
        const int rc = pilco_gp_predict(&pr->dyn, 0, pol.Ds, pr->P, ws + L.xt, ws + L.mean, ws + L.var, 0,
                                        ws + L.pws, L.pws_bytes, stream);
        if (rc) return rc;
    }
    return PILCO_OK;
}

size_t pilco_particles_grad_workspace_bytes(const pilco_particles* pr) {
    if (!pr || !pt_sizes_ok(pr)) return 0;
    const PgWs L = pg_ws_layout(pr, 1);
    return L.pws_bytes ? L.total : 0;
}

int pilco_particles_rollout_grad(const pilco_particles* pr, const pilco_particles_grad* g, pilco_stream_t stream) {
    int rc = pt_check_desc(pr);
    if (rc) return rc;
    rc = pg_check(pr, 1, g);
    if (rc) return rc;
    return pg_run(pr, 1, g, stream);
}

size_t pilco_particles_batch_grad_workspace_bytes(const pilco_particles* pr, int R) {
    if (!pr || !pt_sizes_ok(pr) || !pt_batch_ok(pr->P, R)) return 0;
    const PgWs L = pg_ws_layout(pr, R);
    return L.pws_bytes ? L.total : 0;
}

int pilco_particles_rollout_batch_grad(const pilco_particles* pr, int R, const pilco_particles_grad* g,
                                       pilco_stream_t stream) {
    int rc = pt_check_desc(pr, true);
    if (rc) return rc;
    if (!pt_batch_ok(pr->P, R)) return PILCO_ERR_DIM;
    rc = pg_check(pr, R, g);
    if (rc) return rc;
    return pg_run(pr, R, g, stream);
}

size_t pilco_particles_consistent_workspace_bytes(const pilco_particles* pr) {
    if (!pr || !pt_sizes_ok(pr)) return 0;
    const FsWs L = fs_ws_layout(pr);
    return L.ok && L.pws_bytes ? L.total : 0;
}

// pt_step<0>, fs_predict<0>, fs_cond<0>, pt_step<1>, ..., fs_cond<H-1>, pt_step<H>: pt_step_kernel unchanged, reading
// the step closure (mean, var) fs_cond_kernel leaves
int pilco_particles_rollout_consistent(const pilco_particles* pr, pilco_stream_t stream) {
    int rc = pt_check_desc(pr);
    if (rc) return rc;
    if (!pr->ws) return PILCO_ERR_NULL;
    if ((uintptr_t)pr->ws & 15) return PILCO_ERR_ALIGN;
    const FsWs L = fs_ws_layout(pr);
    if (!L.ok || L.pws_bytes == 0) return PILCO_ERR_DIM;
    if (pr->ws_bytes < L.total) return PILCO_ERR_WORKSPACE;
    rc = fs_predict_prepare();
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    double* ws = (double*)pr->ws;
    const int P = pr->P, H = pr->H, Ds = pr->pol.Ds, D = pr->dyn.D;
    const size_t PD = (size_t)P * D, slot = (size_t)Ds * P * pad64(pr->dyn.n);
    PtDev a = pt_dev(pr);
    a.mean = ws + L.mean; a.var = ws + L.var;
    FsCond c;
    c.P = P; c.H = H; c.D = D; c.Ds = Ds; c.n = pr->dyn.n; c.np = pad64(pr->dyn.n); c.t = 0;
    c.ell = pr->dyn.ell; c.sf2 = pr->dyn.sf2;
    c.xh = ws + L.xh; c.mu = ws + L.mu; c.s2 = ws + L.s2; c.W = ws + L.W; c.Kh = ws + L.Kh;
    c.eps = pr->eps; c.L = ws + L.L; c.mean = ws + L.mean; c.var = ws + L.var;
    const dim3 grid((P + PT_THREADS - 1) / PT_THREADS), cgrid((P + FS_WARPS - 1) / FS_WARPS, Ds);
    for (int t = 0; t <= H; ++t) {
        a.t = t;
        a.xt = ws + L.xh + (size_t)(t < H ? t : 0) * PD;
        launch_hi(pt_step_kernel, grid, dim3(PT_THREADS), 0, st, a);
        CUDA_LAUNCH_CHECK();
        if (t == H) break;
        rc = fs_predict_launch(st, &pr->dyn, P, a.xt, ws + L.mu, ws + L.s2, ws + L.W, ws + L.Kh + (size_t)t * slot,
                               ws + L.pws);
        if (rc) return rc;
        c.t = t;
        launch_hi(fs_cond_kernel, cgrid, dim3(FS_WARPS * 32), 0, st, c);
        CUDA_LAUNCH_CHECK();
    }
    return PILCO_OK;
}

}  // extern "C"
