// particles_mlp.cu -- tanh MLP policies in the particle rollouts (DESIGN.md section 29), the policy class Deep PILCO
// trains on sampled returns:
//   h_1 = tanh(A_1 [x; 1]),  h_2 = tanh(A_2 [h_1; 1])  (L = 2),  z = A_out [h_L; 1],  u = maxa sin(z) (squash) or z
// Only the step kernels and the policy-parameter reduction read the policy (section 28), so the MLP needs:
//   pm_step_kernel    pt_step_kernel with the MLP as the policy (the closure, rewards, x~_t and return in its order)
//   pm_refit_kernel   pr_step_kernel's redraw, then the same work
//   pm_reverse_kernel pg_step_kernel's cotangent algebra with the MLP's input VJP; the activations are recomputed from
//                     the stored policy input, and the step's layer inputs [a_{l-1}; 1] and pre-activation cotangents
//                     d_l go to per-step buffers (feature-major, reused by every step)
//   reduction         per step and layer one batched gemm() (factorize.cu, DMMA) into per-chunk partials
//                     part[r, c] += d_l' [a_{l-1}; 1] over chunk c's rows of restart r; pm_finish_kernel then sums the
//                     chunks in order, over P.  A restart's sums depend on P only, not on R.
// One thread per particle.  The step kernels keep h_1 in registers (fully unrolled over PM_MAXW with width guards), the
// reverse kernel in shared memory; the weights are read from global memory (uniform across a restart's CTA).
#include "particles.cuh"
#include "gemm.cuh"

#define PM_RTHREADS 64                  // pm_reverse_kernel's CTA: h_1 in 32 KB of shared memory

// z [U] at the policy input x (restart r's theta th): h_1 in registers, h_2 streamed into z
__device__ __forceinline__ void pm_forward(const PmNet& m, const double* th, int Ds, int U, const double (&x)[MAXD],
                                           double (&z)[MAXD]) {
    const int w1 = m.w1, wl = m.L == 2 ? m.w2 : w1, ldo = wl + 1;
    const double* Ao = th + m.offo;
    double h1[PM_MAXW];
#pragma unroll
    for (int i = 0; i < PM_MAXW; ++i) {
        h1[i] = 0.0;
        if (i < w1) {
            const double* a = th + i * (Ds + 1);
            double s = a[Ds];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < Ds) s = fma(a[d], x[d], s);
            h1[i] = tanh(s);
        }
    }
#pragma unroll
    for (int j = 0; j < MAXD; ++j) z[j] = j < U ? Ao[j * ldo + wl] : 0.0;
    if (m.L == 1) {
#pragma unroll
        for (int i = 0; i < PM_MAXW; ++i)
            if (i < w1)
#pragma unroll
                for (int j = 0; j < MAXD; ++j) if (j < U) z[j] = fma(Ao[j * ldo + i], h1[i], z[j]);
        return;
    }
    const double* A2 = th + m.off2;
    for (int i = 0; i < m.w2; ++i) {
        const double* a = A2 + i * (w1 + 1);
        double s = a[w1];
#pragma unroll
        for (int k = 0; k < PM_MAXW; ++k) if (k < w1) s = fma(a[k], h1[k], s);
        const double h = tanh(s);
#pragma unroll
        for (int j = 0; j < MAXD; ++j) if (j < U) z[j] = fma(Ao[j * ldo + i], h, z[j]);
    }
}

// pt_step_at with the MLP as the policy: the same code in the same order for everything that is not the policy, so
// the rewards, x~_t and the return are what the linear path computes at the same states
__device__ __forceinline__ void pm_step_at(const PtDev& a, const PmNet& m, int r, size_t row, double* tr,
                                           const double (&x)[MAXD]) {
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
    double z[MAXD];
    pm_forward(m, m.theta + r * m.theta_bs, Ds, U, x, z);
    // output variance 0, as the linear policy: maxa sin(z), sin as sinpi(z / pi) (pt_step_kernel's reason)
#pragma unroll
    for (int j = 0; j < MAXD; ++j) {
        if (j < U) {
            const double u = a.squash ? a.maxa[j] * sinpi(z[j] * PT_INV_PI) : z[j];
            ao[j] = u;
            xo[Ds + j] = u;
        }
    }
}

// grid (ceil(P / 128), R), one thread per particle p of restart r = blockIdx.y: pt_step_kernel's closure of step t-1,
// then pm_step_at
__global__ void __launch_bounds__(PT_THREADS) pm_step_kernel(PtDev a, PmNet m) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= a.P) return;
    const int Ds = a.Ds, t = a.t, H = a.H;
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
    pm_step_at(a, m, r, row, tr, x);
}

// grid (ceil(P / 128), R): pr_step_kernel's redraw x_pt = mu^_t + L^_t xi_{p,t-1}, then pm_step_at
__global__ void __launch_bounds__(PT_THREADS) pm_refit_kernel(PtDev a, PrFwd f, PmNet m) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= a.P) return;
    const int Ds = a.Ds, t = a.t, H = a.H;
    const size_t row = (size_t)r * a.P + p, s = (size_t)(t - 1) * gridDim.y + r;
    const double* mu = f.mu + s * Ds;
    const double* L = f.L + s * Ds * Ds;
    const double* xi = f.xi + ((size_t)p * H + (t - 1)) * Ds;
    double z[MAXD], x[MAXD];
#pragma unroll
    for (int k = 0; k < MAXD; ++k) z[k] = k < Ds ? xi[k] : 0.0;
#pragma unroll
    for (int i = 0; i < MAXD; ++i) {
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k <= i; ++k) if (i < Ds) acc = fma(L[i * Ds + k], z[k], acc);
        x[i] = i < Ds ? mu[i] + acc : 0.0;
    }
    pm_step_at(a, m, r, row, a.traj + (row * (H + 1) + t) * Ds, x);
}

// grid (ceil(P / 64), R), one thread per particle p of restart r = blockIdx.y: step t of the reverse sweep.
// pg_step_kernel's algebra: x_bar_t = x_bar_{t+1} + x~_bar_t[:Ds] + sum_k a_kt grad v_k(x_t) + (d pi / dx)' z_bar_t and
// var_bar_{t-1}; the MLP's VJP (a_l = the layer's activations, a_0 = x):
//   d_out = z_bar_t = x~_bar_t[Ds:] o maxa cos(z)  (squash),  d_l = (A_{l+1}[:, :w_l]' d_{l+1}) o (1 - a_l^2),
//   (d pi / dx)' z_bar_t = A_1[:, :Ds]' d_1
// With x~_bar_t (a.gxt) the step's [a_{l-1}; 1] and d_l go to b's buffers; without it (t = H-1 with no joint or bonus
// term) z_bar_t = 0 and the buffers are not touched (the host skips the step's products).  h_1, then its cotangent,
// is in shared memory (one column per thread, conflict-free); h_1 is read back from the in1 buffer the thread wrote.
__global__ void __launch_bounds__(PM_RTHREADS) pm_reverse_kernel(PgDev a, PmBwd b) {
    PDL_ENTRY();
    __shared__ double sh[PM_MAXW * PM_RTHREADS];
    const int p = blockIdx.x * PM_RTHREADS + threadIdx.x, r = blockIdx.y;
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
    // reward terms at x_t (box: flat almost everywhere, no gradient): pg_step_kernel's code
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
    if (gxt) {
        const PmNet& m = b.net;
        const double* th = m.theta + r * m.theta_bs;
        const int w1 = m.w1, w2 = m.w2, L2 = m.L == 2, wl = L2 ? w2 : w1, ldo = wl + 1;
        const double* A2 = th + m.off2;
        const double* Ao = th + m.offo;
        const size_t RPp = b.RPp, col = (size_t)r * b.Pp + p;
        double* h1 = sh + threadIdx.x;                  // h_1, then its cotangent, at [k PM_RTHREADS]
#pragma unroll
        for (int d = 0; d < MAXD; ++d) if (d < Ds) b.in0[d * RPp + col] = x[d];
        b.in0[Ds * RPp + col] = 1.0;
        for (int i = 0; i < w1; ++i) {                  // pm_forward's order throughout
            const double* ar = th + i * (Ds + 1);
            double s = ar[Ds];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < Ds) s = fma(ar[d], x[d], s);
            const double h = tanh(s);
            h1[i * PM_RTHREADS] = h;
            b.in1[i * RPp + col] = h;
        }
        b.in1[w1 * RPp + col] = 1.0;
        if (L2) {
            for (int i = 0; i < w2; ++i) {
                const double* ar = A2 + i * (w1 + 1);
                double s = ar[w1];
                for (int k = 0; k < w1; ++k) s = fma(ar[k], h1[k * PM_RTHREADS], s);
                b.in2[i * RPp + col] = tanh(s);
            }
            b.in2[w2 * RPp + col] = 1.0;
        }
        const double* hl = L2 ? b.in2 + col : b.in1 + col;
        for (int j = 0; j < U; ++j) {                   // z_j (bias, then the hidden units in order) and d_out,j
            const double* ar = Ao + j * ldo;
            double z = ar[wl];
            for (int i = 0; i < wl; ++i) z = fma(ar[i], hl[i * RPp], z);
            double zbj = gxt[Ds + j];
            // cos(z) as cospi(z / pi): no Payne-Hanek slow path (and its local-memory table), as the forward's sinpi
            if (a.squash) zbj *= a.maxa[j] * cospi(z * PT_INV_PI);
            b.dout[j * RPp + col] = zbj;
        }
        for (int k = 0; k < w1; ++k) h1[k * PM_RTHREADS] = 0.0;     // now the cotangent of h_1
        if (L2) {
            for (int i = 0; i < w2; ++i) {
                double g = 0.0;
                for (int j = 0; j < U; ++j) g = fma(Ao[j * ldo + i], b.dout[j * RPp + col], g);
                const double h = b.in2[i * RPp + col];
                const double d2 = g * (1.0 - h * h);
                b.d2[i * RPp + col] = d2;
                const double* ar = A2 + i * (w1 + 1);
                for (int k = 0; k < w1; ++k) h1[k * PM_RTHREADS] = fma(ar[k], d2, h1[k * PM_RTHREADS]);
            }
        } else {
            for (int k = 0; k < w1; ++k) {
                double g = 0.0;
                for (int j = 0; j < U; ++j) g = fma(Ao[j * ldo + k], b.dout[j * RPp + col], g);
                h1[k * PM_RTHREADS] = g;
            }
        }
        for (int k = 0; k < w1; ++k) {
            const double h = b.in1[k * RPp + col];
            const double d1 = h1[k * PM_RTHREADS] * (1.0 - h * h);
            b.d1[k * RPp + col] = d1;
            const double* ar = th + k * (Ds + 1);
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < Ds) xb[d] = fma(ar[d], d1, xb[d]);
        }
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

// grid (ceil(n_theta / 256) + 1, R), 256 threads: gtheta[r, i] = (sum_c part[r, c, i]) / P, chunks in order; the last
// CTA of restart r = blockIdx.y the mean return, pg_param_kernel's value CTA
__global__ void __launch_bounds__(256) pm_finish_kernel(int P, int nc, int n_theta, const double* part,
                                                        const double* ret, double* gtheta, double* value) {
    PDL_ENTRY();
    __shared__ double red[8], out[1];
    const int r = blockIdx.y, tid = threadIdx.x;
    const double invP = 1.0 / P;
    if ((int)blockIdx.x == gridDim.x - 1) {
        double v[1] = {0.0};
        for (int p = tid; p < P; p += 256) v[0] += ret[(size_t)r * P + p];
        pg_block_sum<1>(v, red, out);
        if (tid == 0) value[r] = out[0] * invP;
        return;
    }
    const int i = blockIdx.x * 256 + tid;
    if (i >= n_theta) return;
    const double* pr = part + (size_t)r * nc * n_theta + i;
    double s = 0.0;
    for (int c = 0; c < nc; ++c) s += pr[(size_t)c * n_theta];
    gtheta[(size_t)r * n_theta + i] = s * invP;
}

int pm_step_launch(cudaStream_t st, dim3 grid, const PtDev& a, const PmNet& m) {
    launch_hi(pm_step_kernel, grid, dim3(PT_THREADS), 0, st, a, m);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int pm_refit_launch(cudaStream_t st, dim3 grid, const PtDev& a, const PrFwd& f, const PmNet& m) {
    launch_hi(pm_refit_kernel, grid, dim3(PT_THREADS), 0, st, a, f, m);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int pm_reverse_launch(cudaStream_t st, dim3 grid, const PgDev& a, const PmBwd& b) {
    launch_hi(pm_reverse_kernel, dim3((a.P + PM_RTHREADS - 1) / PM_RTHREADS, grid.y), dim3(PM_RTHREADS), 0, st, a, b);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int pm_finish_launch(cudaStream_t st, int R, int P, int nc, int n_theta, const double* part, const double* ret,
                     double* gtheta, double* value) {
    launch_hi(pm_finish_kernel, dim3((n_theta + 255) / 256 + 1, R), dim3(256), 0, st, P, nc, n_theta, part, ret, gtheta,
              value);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}
