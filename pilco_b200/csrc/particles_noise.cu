// particles_noise.cu -- the particle rollouts with measurement noise at the policy's input (DESIGN.md section 23):
//   z_t = x_t + sqrt(v) o nu_t,  u_t = squash(pi(phi(z_t))),  x~_t = [phi(x_t), u_t],
//   x_{t+1} = x_t + mu(x~_t) + sqrt(max(var(x~_t), 0)) o eps_t
// nu [P,H,E] is the caller's standard normals, shared by the restarts like eps.  phi is section 20's map (the identity
// with A = 0).  The state stays raw; the state reward terms see x_t, the joint terms x~_t.
// These kernels replace pa_step_kernel and pa_policy_bwd / pa_state_bwd in the noisy path; every other launch of
// particles.cu is reused with its pointers and widths.  They live in their own translation unit so that the existing
// kernels keep their register allocation.
// The forward writes phi(x_t) and phi(z_t) once each (gradients: to their histories); the reverse step reads those
// histories, so both directions see the same sin and cos bits.
#include "particles.cuh"

// grid (ceil(P / 128), R), one thread per particle p of restart r = blockIdx.y: close step t-1 in E, write traj[:, t],
// the state terms at x_t; phi(z_t) (z gathered element by element from the raw row and nu) through x~_t[:Dh] into
// registers, then phi(x_t) to x~_t[:Dh]; the policy at phi(z_t) to act and x~_t[Dh:].  At t = H the return, as
// pt_step_kernel.  The minimum of 4 CTAs per SM caps it at 128 registers; left free, ptxas settles at 96 and spills
// a row offset around the step closure's sqrt slow-path calls.
__global__ void __launch_bounds__(PT_THREADS, 4) pn_step_kernel(PnStep a) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= a.P) return;
    const int E = a.E, Dh = a.Ds, U = a.U, D = Dh + U, t = a.t, H = a.H;
    const size_t row = (size_t)r * a.P + p;
    double* tr = a.traj + (row * (H + 1) + t) * E;
    double x[MAXD];
    if (t == 0) {
#pragma unroll
        for (int d = 0; d < MAXD; ++d) x[d] = d < E ? a.x0[(size_t)p * E + d] : 0.0;
    } else {                                            // close step t-1
        const double* xp = tr - E;
        const double* mu = a.mean + row * E;
        const double* var = a.var + row * E;
        const double* ep = a.eps + ((size_t)p * H + (t - 1)) * E;
#pragma unroll
        for (int d = 0; d < MAXD; ++d) {
            if (d < E) {
                const double v = var[d];
                x[d] = fma(sqrt(v < 0.0 ? 0.0 : v), ep[d], xp[d] + mu[d]);      // NaN stays NaN
            } else x[d] = 0.0;
        }
    }
#pragma unroll
    for (int d = 0; d < MAXD; ++d) if (d < E) tr[d] = x[d];
    const size_t ph = row * H;
    if (t == H) {                                       // return: step order, as pt_step_kernel
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
    double rew = 0.0, risk = 0.0;                       // the state terms at the raw x_t
    for (int k = 0; k < a.n_rewards; ++k) {
        const pilco_reward_term& rt = a.rewards[k];
        const double v = pt_reward_value(rt, x, tr, E);
        if (rt.channel == PILCO_CHANNEL_MULT) risk = fma(rt.coef, v, risk);
        else rew = fma(rt.coef, v, rew);
    }
    a.step_reward[ph + t] = rew;
    a.step_risk[ph + t] = risk;
    // phi(z_t) then phi(x_t), column k from the raw row (indexed reads stay in global memory, not in registers);
    // z_i = fma(sqrt(v_i), nu_i, x_i), so v_i = 0 gives z_i = x_i whatever nu_i
    double* xo = a.xt + row * D;
    double* fo = a.phi ? a.phi + (row * (H + 1) + t) * Dh : nullptr;
    double* fz = a.phiz ? a.phiz + (row * (H + 1) + t) * Dh : nullptr;
    const double* nu = a.nz.nu + ((size_t)p * H + t) * E;
    const int np = a.tm.np;
    for (int k = 0; k < Dh; ++k) {
        const int q = k - np, i = q < 0 ? a.tm.pass[k] : a.tm.ang[q >> 1];
        double f = fma(a.nz.sv[i], nu[i], tr[i]);
        if (q >= 0) {
            double sn, cs;
            sincospi(f * PT_INV_PI, &sn, &cs);
            f = (q & 1) ? cs : sn;
        }
        xo[k] = f;
        if (fz) fz[k] = f;
    }
    double z[MAXD];
#pragma unroll
    for (int d = 0; d < MAXD; ++d) z[d] = d < Dh ? xo[d] : 0.0;
    for (int k = 0; k < Dh; ++k) {
        const int q = k - np;
        double f = tr[q < 0 ? a.tm.pass[k] : a.tm.ang[q >> 1]];
        if (q >= 0) {
            double sn, cs;
            sincospi(f * PT_INV_PI, &sn, &cs);
            f = (q & 1) ? cs : sn;
        }
        xo[k] = f;
        if (fo) fo[k] = f;
    }
    double* ao = a.act + (ph + t) * U;
    // the policy at z = phi(z_t): pa_step_kernel's code and order
    const double su = a.pol_kind == PILCO_POLICY_RBF ? PT_RBF_VAR : 0.0;
    for (int j = 0; j < U; ++j) {
        double u;
        if (a.pol_kind == PILCO_POLICY_LINEAR) {
            const double* W = a.W + r * a.W_bs;
            u = a.b[r * a.b_bs + j];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < Dh) u = fma(W[j * Dh + d], z[d], u);
        } else {
            const double* ell = a.ell + r * a.ell_bs;
            double il[MAXD];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) il[d] = d < Dh ? 1.0 / ell[j * Dh + d] : 0.0;
            const double sf2 = a.sf2[r * a.sf2_bs + j];
            const double* be = a.beta + r * a.beta_bs + (size_t)j * a.bf;
            const double* C = a.C + r * a.C_bs;
            u = 0.0;
            for (int i = 0; i < a.bf; ++i) {
                const double* c = C + (size_t)i * Dh;
                double d2 = 0.0;
#pragma unroll
                for (int d = 0; d < MAXD; ++d) if (d < Dh) { const double q = (z[d] - c[d]) * il[d]; d2 = fma(q, q, d2); }
                u = fma(sf2 * exp(-0.5 * d2), be[i], u);
            }
        }
        if (a.squash) u = a.maxa[j] * exp(-0.5 * su) * sinpi(u * PT_INV_PI);
        ao[j] = u;
        xo[Dh + j] = u;
    }
}

// Reverse step t, first half: the policy at phi(z_t) (read from the phi(z) history).
//   z_bar_t = x~_bar_t[Dh:] o maxa e^{-su/2} cos(.) (when squashed),  phi_bar_z,t = (d pi / d phi |phi(z_t))' z_bar_t
// phi_bar_z,t goes to its own slot; phi_bar_x,t = x~_bar_t[:Dh] is left where it is.  gxt = NULL (t = H-1 without
// joint terms): z_bar_t = 0, nothing else.
__global__ void __launch_bounds__(PT_THREADS) pn_policy_bwd_kernel(PnBwd a) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= a.P) return;
    const int Dh = a.Ds, U = a.U, t = a.t, H = a.H;
    const size_t row = (size_t)r * a.P + p;
    double* zb = a.zbar + (row * H + t) * U;
    if (!a.gxt) {
        for (int j = 0; j < U; ++j) zb[j] = 0.0;
        return;
    }
    const double* gxt = a.gxt + row * (Dh + U);
    const double* fg = a.phiz + (row * (H + 1) + t) * Dh;
    double z[MAXD], fb[MAXD];
#pragma unroll
    for (int d = 0; d < MAXD; ++d) {
        z[d] = d < Dh ? fg[d] : 0.0;
        fb[d] = 0.0;
    }
    // the action recomputed in the forward's order (pn_step_kernel), with the Jacobian row as pa_policy_bwd_kernel
    const double su = a.pol_kind == PILCO_POLICY_RBF ? PT_RBF_VAR : 0.0;
    for (int j = 0; j < U; ++j) {
        double jx[MAXD], u;
        if (a.pol_kind == PILCO_POLICY_LINEAR) {
            const double* W = a.W + r * a.W_bs;
            u = a.b[r * a.b_bs + j];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) {
                jx[d] = d < Dh ? W[j * Dh + d] : 0.0;
                if (d < Dh) u = fma(W[j * Dh + d], z[d], u);
            }
        } else {                                        // d u_j / d phi = sum_i beta_ji k_ji (c_i - phi) / ell_j^2
            const double* ell = a.ell + r * a.ell_bs;
            double il[MAXD];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) { il[d] = d < Dh ? 1.0 / ell[j * Dh + d] : 0.0; jx[d] = 0.0; }
            const double sf2 = a.sf2[r * a.sf2_bs + j];
            const double* be = a.beta + r * a.beta_bs + (size_t)j * a.bf;
            const double* C = a.C + r * a.C_bs;
            u = 0.0;
            for (int i = 0; i < a.bf; ++i) {
                const double* c = C + (size_t)i * Dh;
                double d2 = 0.0;
#pragma unroll
                for (int d = 0; d < MAXD; ++d) if (d < Dh) { const double q = (z[d] - c[d]) * il[d]; d2 = fma(q, q, d2); }
                const double kb = sf2 * exp(-0.5 * d2);
                u = fma(kb, be[i], u);
                const double f = kb * be[i];
#pragma unroll
                for (int d = 0; d < MAXD; ++d) if (d < Dh) jx[d] = fma(f, (c[d] - z[d]) * (il[d] * il[d]), jx[d]);
            }
        }
        double zbj = gxt[Dh + j];
        if (a.squash) zbj *= a.maxa[j] * exp(-0.5 * su) * cospi(u * PT_INV_PI);
        zb[j] = zbj;
#pragma unroll
        for (int d = 0; d < MAXD; ++d) if (d < Dh) fb[d] = fma(zbj, jx[d], fb[d]);
    }
    double* fo = a.phibz + row * Dh;
#pragma unroll
    for (int d = 0; d < MAXD; ++d) if (d < Dh) fo[d] = fb[d];
}

// Reverse step t, second half, in the raw state (E).  dz/dx = I, so the state takes both feature Jacobians:
//   x_bar_t = x_bar_{t+1} + J_phi(x_t)' phi_bar_x,t + J_phi(z_t)' phi_bar_z,t + sum_k a_kt grad v_k(x_t)
// J_phi(y)' f: a pass-through dimension takes its column; angle a takes cos y_a f_sin - sin y_a f_cos, with sin and cos
// the forward's (the phi(x) and phi(z) histories).  Then the cotangents of step t-1's predict outputs, as
// pa_state_bwd_kernel.  gxt = NULL: x_bar_{t+1} and both feature cotangents are 0.
__global__ void __launch_bounds__(PT_THREADS) pn_state_bwd_kernel(PnBwd a) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= a.P) return;
    const int E = a.E, Dh = a.Ds, U = a.U, t = a.t, H = a.H;
    const size_t row = (size_t)r * a.P + p;
    const double* xg = a.traj + (row * (H + 1) + t) * E;
    const double* fb = a.gxt ? a.gxt + row * (Dh + U) : nullptr;
    const double* zb = a.phibz + row * Dh;
    const double* fg = a.phi + (row * (H + 1) + t) * Dh;
    const double* zg = a.phiz + (row * (H + 1) + t) * Dh;
    double x[MAXD], xb[MAXD];
#pragma unroll
    for (int d = 0; d < MAXD; ++d) {
        x[d] = d < E ? xg[d] : 0.0;
        xb[d] = 0.0;
        if (d < E && fb) {
            const int k = a.tm.pos[d];                  // an angle: its sine column; the cosine column follows
            const double v = a.tm.isang[d] ? fma(fg[k + 1], fb[k], -(fg[k] * fb[k + 1])) : fb[k];
            const double w = a.tm.isang[d] ? fma(zg[k + 1], zb[k], -(zg[k] * zb[k + 1])) : zb[k];
            xb[d] = a.gx[row * E + d] + v + w;
        }
    }
    double wmult = 0.0;
    if (a.n_mult > 0) {                                 // mult_mu prod_{s != t} (1 - risk_s), as pg_step_kernel
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
            for (int d = 0; d < MAXD; ++d) if (d < E) xb[d] = fma(w, rt.W[d], xb[d]);
            continue;
        }
        double v[MAXD], gv[MAXD];                       // exp(-0.5 v' W v), v = x - t: gradient -value (W + W') v / 2
#pragma unroll
        for (int i = 0; i < MAXD; ++i) v[i] = i < E ? x[i] - rt.t[i] : 0.0;
        double quad = 0.0;
#pragma unroll
        for (int i = 0; i < MAXD; ++i) {
            gv[i] = 0.0;
            if (i < E) {
                double wy = 0.0, wty = 0.0;
#pragma unroll
                for (int k2 = 0; k2 < MAXD; ++k2)
                    if (k2 < E) { wy = fma(rt.W[i * E + k2], v[k2], wy); wty = fma(rt.W[k2 * E + i], v[k2], wty); }
                quad = fma(v[i], wy, quad);
                gv[i] = wy + wty;
            }
        }
        const double f = -0.5 * w * exp(-0.5 * quad);
#pragma unroll
        for (int d = 0; d < MAXD; ++d) if (d < E) xb[d] = fma(f, gv[d], xb[d]);
    }
#pragma unroll
    for (int d = 0; d < MAXD; ++d) if (d < E) a.gx[row * E + d] = xb[d];
    if (t > 0) {                                        // cotangents of step t-1's predict outputs
        const double* vp = a.var_prev + row * E;
        const double* ep = a.eps + ((size_t)p * H + (t - 1)) * E;
#pragma unroll
        for (int d = 0; d < MAXD; ++d) {
            if (d < E) {
                const double v = vp[d];
                a.gvar[row * E + d] = v > 0.0 ? xb[d] * ep[d] / (2.0 * sqrt(v)) : 0.0;
            }
        }
    }
}

int pn_step_launch(cudaStream_t st, dim3 grid, const PnStep& a) {
    launch_hi(pn_step_kernel, grid, dim3(PT_THREADS), 0, st, a);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int pn_reverse_launch(cudaStream_t st, dim3 grid, const PnBwd& a) {
    launch_hi(pn_policy_bwd_kernel, grid, dim3(PT_THREADS), 0, st, a);
    CUDA_LAUNCH_CHECK();
    launch_hi(pn_state_bwd_kernel, grid, dim3(PT_THREADS), 0, st, a);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}
