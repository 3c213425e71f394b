// particles_resample.cu -- Gaussian-resampled particle rollouts (Deep PILCO's refit; DESIGN.md section 26):
// pilco_particles_resampled_rollout and pilco_particles_resampled_grad_rollout.  Per restart r over its P particles and
// step t >= 1 (x_0 = x0, no refit at t = 0):
//   x'_pt = x_{p,t-1} + mu(x~_{p,t-1}) + sqrt(max(var, 0)) o eps_{p,t-1}        pt_step_kernel's closure, same fma order
//   mu^_t = (1/P) sum_p x'_pt,  S^_t = 1/(P-1) sum_p (x'_pt - mu^_t)(x'_pt - mu^_t)'        two-pass, fixed order
//   L^_t  = pr_chol(S^_t) (resample_math.cuh: a column whose pivot is <= 1e-12 S^_jj is zeroed)
//   x_pt  = mu^_t + L^_t xi_{p,t-1}
// and the rewards, the policy and x~_t are evaluated at the refitted x_pt, as pt_step_kernel evaluates them.
// Launches of step t >= 1 (in place of pt_step<t>): pr_close (per particle), pr_moments (one CTA per restart),
// pr_step (per particle: the redraw and pt_step_kernel's work, pt_step_at).  Reverse stage of step t = H-1 .. 1, after
// the reverse step kernel: pr_adjoint (one CTA per restart: mu_bar = sum_p y_bar_p, L_bar = tril(sum_p y_bar_p xi_p'),
// the Cholesky reverse A = d value / d S^ on its lower triangle) and pr_scatter (per particle:
// x'_bar_p = mu_bar / P + (A + A')(x'_p - mu^) / (P-1), gx <- x'_bar_p, gvar <- x'_bar_p o eps_{t-1} / (2 s_{t-1})).
// Every sum over a restart's particles is fixed-order (thread q takes p = q, q + 256, ..., then pg_block_sum), so a
// restart's results do not depend on R.
#include "particles.cuh"
#include "resample_math.cuh"

// rows of a [P, ld] array (restart base already applied), minus the shared-memory centre c when c is not NULL
struct PrRows {
    const double* x; long long ld; const double* c;
};

// S[i Ds + j] (j <= i) = sum_p a_pi b_pj over the P rows, fixed order; four rows of S per pass so the accumulators stay
// in registers (every index below is a compile-time constant), each pass one pg_block_sum.  red [64 8], out [64].
__device__ __forceinline__ void pr_tril_sums(int P, int Ds, PrRows A, PrRows B, double* red, double* out, double* S) {
#pragma unroll
    for (int i0 = 0; i0 < MAXD; i0 += 4) {
        if (i0 < Ds) {
            double acc[4 * MAXD];
#pragma unroll
            for (int c = 0; c < 4 * MAXD; ++c) acc[c] = 0.0;
            for (int p = threadIdx.x; p < P; p += 256) {
                const double* ra = A.x + (size_t)p * A.ld;
                const double* rb = B.x + (size_t)p * B.ld;
                double va[4], vb[MAXD];
#pragma unroll
                for (int ii = 0; ii < 4; ++ii) {
                    const int i = i0 + ii;
                    va[ii] = i < Ds ? (A.c ? ra[i] - A.c[i] : ra[i]) : 0.0;
                }
#pragma unroll
                for (int j = 0; j < MAXD; ++j) vb[j] = (j < Ds && j < i0 + 4) ? (B.c ? rb[j] - B.c[j] : rb[j]) : 0.0;
#pragma unroll
                for (int ii = 0; ii < 4; ++ii)
#pragma unroll
                    for (int j = 0; j <= i0 + ii; ++j) acc[ii * MAXD + j] = fma(va[ii], vb[j], acc[ii * MAXD + j]);
            }
            pg_block_sum<4 * MAXD>(acc, red, out);
            for (int c = threadIdx.x; c < 4 * MAXD; c += 256) {
                const int i = i0 + c / MAXD, j = c % MAXD;
                if (i < Ds && j <= i) S[i * Ds + j] = out[c];
            }
        }
    }
    __syncthreads();
}

// sum_p x_p over the P rows -> out[0..Ds), fixed order
__device__ __forceinline__ void pr_vec_sum(int P, int Ds, PrRows A, double* red, double* out) {
    double v[MAXD];
#pragma unroll
    for (int d = 0; d < MAXD; ++d) v[d] = 0.0;
    for (int p = threadIdx.x; p < P; p += 256) {
        const double* ra = A.x + (size_t)p * A.ld;
#pragma unroll
        for (int d = 0; d < MAXD; ++d) if (d < Ds) v[d] += ra[d];
    }
    pg_block_sum<MAXD>(v, red, out);
}

// grid (ceil(P / 128), R): x'_t of particle p of restart r = blockIdx.y into its slot of the x' history
__global__ void __launch_bounds__(PT_THREADS) pr_close_kernel(PtDev a, PrFwd f) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x;
    if (p >= a.P) return;
    const int Ds = a.Ds, t = a.t, H = a.H;
    const size_t row = (size_t)blockIdx.y * a.P + p, T = (size_t)gridDim.y * a.P;
    const double* xp = a.traj + (row * (H + 1) + t - 1) * Ds;
    const double* mu = a.mean + row * Ds;
    const double* var = a.var + row * Ds;
    const double* ep = a.eps + ((size_t)p * H + (t - 1)) * Ds;
    double* xo = f.xp + ((size_t)(t - 1) * T + row) * Ds;
    for (int d = 0; d < Ds; ++d) {
        const double v = var[d];
        xo[d] = fma(sqrt(v < 0.0 ? 0.0 : v), ep[d], xp[d] + mu[d]);          // NaN stays NaN
    }
}

// the moments of one restart's rows: x [P,Ds] at x + r rs (rs = 0: x0, shared by the restarts); the sample mean and
// unbiased covariance of step t into step_mean / step_cov (when given) and, for t >= 1, mu^ and L^ into slot t-1
struct PrMom {
    int P, Ds, t, H;
    const double* x; long long rs;
    double* mu; double* L;
    double* step_mean; double* step_cov;
};

// grid (R), 256 threads: restart r = blockIdx.x
__global__ void __launch_bounds__(256) pr_moments_kernel(PrMom m) {
    PDL_ENTRY();
    __shared__ double red[4 * MAXD * 8], out[4 * MAXD], c[MAXD], S[MAXD * MAXD], Lf[MAXD * MAXD];
    const int P = m.P, Ds = m.Ds, r = blockIdx.x, tid = threadIdx.x;
    const double* x = m.x + (size_t)r * m.rs;
    pr_vec_sum(P, Ds, {x, Ds, nullptr}, red, out);
    if (tid < Ds) c[tid] = out[tid] / P;
    __syncthreads();
    pr_tril_sums(P, Ds, {x, Ds, c}, {x, Ds, c}, red, out, S);
    if (tid != 0) return;
    const double inv = 1.0 / (P - 1);
    for (int i = 0; i < Ds; ++i)
        for (int j = 0; j <= i; ++j) S[j * Ds + i] = S[i * Ds + j] = S[i * Ds + j] * inv;
    const size_t o = (size_t)r * (m.H + 1) + m.t;
    if (m.step_mean) for (int i = 0; i < Ds; ++i) m.step_mean[o * Ds + i] = c[i];
    if (m.step_cov) for (int i = 0; i < Ds * Ds; ++i) m.step_cov[o * Ds * Ds + i] = S[i];
    if (!m.L) return;
    pr_chol(S, Lf, Ds);
    const size_t s = (size_t)(m.t - 1) * gridDim.x + r;
    for (int i = 0; i < Ds; ++i) m.mu[s * Ds + i] = c[i];
    for (int i = 0; i < Ds * Ds; ++i) m.L[s * Ds * Ds + i] = Lf[i];
}

// grid (ceil(P / 128), R): x_pt = mu^_t + L^_t xi_{p,t-1} for particle p of restart r = blockIdx.y, then pt_step_at
__global__ void __launch_bounds__(PT_THREADS) pr_step_kernel(PtDev a, PrFwd f) {
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
    pt_step_at(a, r, row, a.traj + (row * (H + 1) + t) * Ds, x);
}

// grid (R), 256 threads: restart r = blockIdx.x's mu_bar / P and (A + A') / (P-1) at step t into sc
__global__ void __launch_bounds__(256) pr_adjoint_kernel(PrBwd b) {
    PDL_ENTRY();
    __shared__ double red[4 * MAXD * 8], out[4 * MAXD], mb[MAXD], Lb[MAXD * MAXD], Lf[MAXD * MAXD], Sb[MAXD * MAXD];
    const int P = b.P, Ds = b.Ds, H = b.H, r = blockIdx.x, tid = threadIdx.x;
    const double* gx = b.gx + (size_t)r * P * Ds;
    pr_vec_sum(P, Ds, {gx, Ds, nullptr}, red, out);
    if (tid < Ds) mb[tid] = out[tid];
    for (int i = tid; i < Ds * Ds; i += 256) Lb[i] = 0.0;
    __syncthreads();
    pr_tril_sums(P, Ds, {gx, Ds, nullptr}, {b.xi + (size_t)(b.t - 1) * Ds, (long long)H * Ds, nullptr}, red, out, Lb);
    if (tid != 0) return;
    const size_t s = (size_t)(b.t - 1) * gridDim.x + r;
    for (int i = 0; i < Ds * Ds; ++i) Lf[i] = b.L[s * Ds * Ds + i];
    pr_chol_bwd(Lf, Lb, Sb, Ds);
    double* sc = b.sc + (size_t)r * (Ds + Ds * Ds);
    for (int i = 0; i < Ds; ++i) sc[i] = mb[i] / P;
    const double inv = 1.0 / (P - 1);
    for (int i = 0; i < Ds; ++i)                        // Sb's upper triangle is 0
        for (int j = 0; j < Ds; ++j) sc[Ds + i * Ds + j] = (Sb[i * Ds + j] + Sb[j * Ds + i]) * inv;
}

// grid (ceil(P / 128), R): particle p of restart r = blockIdx.y: x'_bar = mu_bar / P + (A + A')(x' - mu^) / (P-1)
// into gx, and the cotangent of var_{t-1} (pg_step_kernel's formula at x'_bar) into gvar
__global__ void __launch_bounds__(PT_THREADS) pr_scatter_kernel(PrBwd b) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= b.P) return;
    const int Ds = b.Ds, t = b.t;
    const size_t row = (size_t)r * b.P + p, T = (size_t)gridDim.y * b.P, s = (size_t)(t - 1) * gridDim.y + r;
    const double* xp = b.xp + ((size_t)(t - 1) * T + row) * Ds;
    const double* mu = b.mu + s * Ds;
    const double* sc = b.sc + (size_t)r * (Ds + Ds * Ds);
    double c[MAXD];
#pragma unroll
    for (int j = 0; j < MAXD; ++j) c[j] = j < Ds ? xp[j] - mu[j] : 0.0;
    const double* vp = b.var_prev + row * Ds;
    const double* ep = b.eps + ((size_t)p * b.H + (t - 1)) * Ds;
#pragma unroll
    for (int i = 0; i < MAXD; ++i) {
        if (i < Ds) {
            double g = sc[i];
#pragma unroll
            for (int j = 0; j < MAXD; ++j) if (j < Ds) g = fma(sc[Ds + i * Ds + j], c[j], g);
            b.gx[row * Ds + i] = g;
            const double v = vp[i];
            b.gvar[row * Ds + i] = v > 0.0 ? g * ep[i] / (2.0 * sqrt(v)) : 0.0;
        }
    }
}

int pr_step_launch(cudaStream_t st, dim3 grid, const PtDev& a, const PrFwd& f, const PmNet* net) {
    const int R = grid.y, t = a.t;
    PrMom m;
    m.P = f.P; m.Ds = f.Ds; m.t = t; m.H = f.H;
    m.step_mean = f.step_mean; m.step_cov = f.step_cov;
    if (t == 0) {                                       // the moments of x0, shared by the restarts
        if (!f.step_mean && !f.step_cov) return PILCO_OK;
        m.x = f.x0; m.rs = 0; m.mu = m.L = nullptr;
        launch_hi(pr_moments_kernel, dim3(R), dim3(256), 0, st, m);
        CUDA_LAUNCH_CHECK();
        return PILCO_OK;
    }
    launch_hi(pr_close_kernel, grid, dim3(PT_THREADS), 0, st, a, f);
    CUDA_LAUNCH_CHECK();
    m.x = f.xp + (size_t)(t - 1) * R * f.P * f.Ds; m.rs = (long long)f.P * f.Ds; m.mu = f.mu; m.L = f.L;
    launch_hi(pr_moments_kernel, dim3(R), dim3(256), 0, st, m);
    CUDA_LAUNCH_CHECK();
    if (net) return pm_refit_launch(st, grid, a, f, *net);
    launch_hi(pr_step_kernel, grid, dim3(PT_THREADS), 0, st, a, f);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int pr_reverse_launch(cudaStream_t st, dim3 grid, const PrBwd& b) {
    launch_hi(pr_adjoint_kernel, dim3(grid.y), dim3(256), 0, st, b);
    CUDA_LAUNCH_CHECK();
    launch_hi(pr_scatter_kernel, grid, dim3(PT_THREADS), 0, st, b);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}
