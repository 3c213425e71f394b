// particles_features.cu -- function-sample particle rollouts in time linear in the horizon (DESIGN.md section 30):
// each particle and dynamics output carries ONE function drawn as a random-feature prior plus an exact data update
// (the decoupled, "pathwise-conditioned" sampler of Wilson et al. 2020),
//   omega_ei = zeta_ei / ell_e,   phi_e(x) = sqrt(sf2_e / F) [cos(omega_e x); sin(omega_e x)]   (2F features)
//   v_pe = beta_e - iK_e (Phi_e(X) w_pe + sqrt(sn2_e) eps_pe)
//   f_pe(x~) = phi_e(x~)' w_pe + sum_j sf2_e exp(-0.5 |(x~ - X_j) / ell_e|^2) v_pe,j
// A function sample is deterministic at a given input, so each step hands the unchanged step kernels mean = f(x~_t) and
// var = 0 where the predict (or fs_cond_kernel) would have left its mean and variance:
//   pilco_particles_features_draw   omega, Phi_e(X) (pf_omega_kernel, pf_phi_kernel), R = Phi W (gemm), R += sqrt(sn2)
//                                   eps and v = beta (pf_prep_kernel), v -= R iK (gemm): once per set of normals
//   pf_eval_kernel                  one warp per (row, output): f at x~_t, in place of the predict
//   pf_vjp_kernel                   one warp per row: x~_bar = sum_e m_bar_e d f_e / d x~, outputs in order
// Each kernel reads w and v at the particle p of its row r P + p (the restarts share the draws), so a particle's
// outputs depend neither on P nor on its row.  sin and cos are sincospi(x / pi): its argument reduction is exact, so no
// Payne-Hanek table lands in local memory.
#include <cmath>
#include "particles.cuh"
#include "gemm.cuh"

#define PF_WARPS 8                      // rows per CTA of the evaluation and VJP kernels
#define PF_CH    128                    // frequencies or centres staged in shared memory per chunk

// one chunk of PF_CH rows of a row-major [., D] array, transposed so that lane i reads s[d][i] without conflicts
// (every thread of the CTA takes part; rows past cnt are not read)
__device__ __forceinline__ void pf_stage(double (&s)[MAXD][PF_CH + 1], const double* src, int cnt, int D) {
    __syncthreads();                                    // the previous chunk is consumed
    for (int q = threadIdx.x; q < cnt * D; q += PF_WARPS * 32) s[q % D][q / D] = src[q];
    __syncthreads();
}

// f_e at x (all lanes: the same bits) and, with GRAD, each lane's share of m_bar d f_e / d x added to g.  Every lane of
// every warp of the CTA calls it (the staging synchronises the CTA); valid = false skips the loads of a padding row.
template <bool GRAD>
__device__ __forceinline__ double pf_output(const PfDev& a, int e, int p, bool valid, const double (&x)[MAXD],
                                            double mbar, double (&s)[MAXD][PF_CH + 1], double (&g)[MAXD]) {
    const int lane = threadIdx.x & 31, D = a.D, F = a.F, n = a.n;
    const double sf2 = a.sf2[e], sc = sqrt(sf2 / F);
    const double* wc = a.w + ((size_t)p * a.E + e) * 2 * F;
    const double* vp = a.v + ((size_t)p * a.E + e) * n;
    double acc = 0.0;
    for (int i0 = 0; i0 < F; i0 += PF_CH) {             // phi_e(x)' w: cos(omega x) w_c + sin(omega x) w_s
        const int cnt = F - i0 < PF_CH ? F - i0 : PF_CH;
        pf_stage(s, a.omega + ((size_t)e * F + i0) * D, cnt, D);
        if (!valid) continue;
        for (int i = lane; i < cnt; i += 32) {
            double arg = 0.0;
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < D) arg = fma(s[d][i], x[d], arg);
            double sn, cs;
            sincospi(arg * PT_INV_PI, &sn, &cs);
            const double c = wc[i0 + i], si = wc[F + i0 + i];
            acc = fma(sc * cs, c, acc);
            acc = fma(sc * sn, si, acc);
            if (GRAD) {
                const double gd = mbar * sc * fma(cs, si, -sn * c);
#pragma unroll
                for (int d = 0; d < MAXD; ++d) if (d < D) g[d] = fma(gd, s[d][i], g[d]);
            }
        }
    }
    double il[MAXD];
#pragma unroll
    for (int d = 0; d < MAXD; ++d) il[d] = d < D ? 1.0 / a.ell[(size_t)e * D + d] : 0.0;
    for (int j0 = 0; j0 < n; j0 += PF_CH) {             // k(x, X) v
        const int cnt = n - j0 < PF_CH ? n - j0 : PF_CH;
        pf_stage(s, a.X + (size_t)j0 * D, cnt, D);
        if (!valid) continue;
        for (int j = lane; j < cnt; j += 32) {
            double d2 = 0.0;
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < D) { const double q = (x[d] - s[d][j]) * il[d]; d2 = fma(q, q, d2); }
            const double kv = sf2 * exp(-0.5 * d2) * vp[j0 + j];
            acc += kv;
            if (GRAD) {
                const double gk = mbar * kv;
#pragma unroll
                for (int d = 0; d < MAXD; ++d) if (d < D) g[d] = fma(gk, (s[d][j] - x[d]) * (il[d] * il[d]), g[d]);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);      // fixed butterfly
    return acc;
}

// x~_t of row `row` into x (0 beyond D)
__device__ __forceinline__ void pf_load_x(const PfDev& a, size_t row, bool valid, double (&x)[MAXD]) {
#pragma unroll
    for (int d = 0; d < MAXD; ++d) x[d] = valid && d < a.D ? a.xh[row * a.D + d] : 0.0;
}

// grid (ceil(T / PF_WARPS), E), one warp per (row, output e = blockIdx.y): mean = f_e(x~_t), var = 0
__global__ void __launch_bounds__(PF_WARPS * 32) pf_eval_kernel(PfDev a) {
    PDL_ENTRY();
    __shared__ double s[MAXD][PF_CH + 1];
    const long long rw = (long long)blockIdx.x * PF_WARPS + (threadIdx.x >> 5);
    const bool valid = rw < a.T;
    const size_t row = valid ? (size_t)rw : 0;
    const int e = blockIdx.y, p = (int)(row % a.P);
    double x[MAXD], g[MAXD];
    pf_load_x(a, row, valid, x);
    const double f = pf_output<false>(a, e, p, valid, x, 0.0, s, g);
    if (valid && (threadIdx.x & 31) == 0) {
        a.mean[row * a.E + e] = f;
        a.var[row * a.E + e] = 0.0;
    }
}

// grid ceil(T / PF_WARPS), one warp per row: x~_bar = sum_e m_bar_e d f_e / d x~ over e in order, each lane's share
// summed by the fixed butterfly per dimension
__global__ void __launch_bounds__(PF_WARPS * 32) pf_vjp_kernel(PfDev a) {
    PDL_ENTRY();
    __shared__ double s[MAXD][PF_CH + 1];
    const long long rw = (long long)blockIdx.x * PF_WARPS + (threadIdx.x >> 5);
    const bool valid = rw < a.T;
    const size_t row = valid ? (size_t)rw : 0;
    const int p = (int)(row % a.P);
    double x[MAXD], g[MAXD];
    pf_load_x(a, row, valid, x);
#pragma unroll
    for (int d = 0; d < MAXD; ++d) g[d] = 0.0;
    for (int e = 0; e < a.E; ++e) {
        const double mbar = valid ? a.gmean[row * a.E + e] : 0.0;
        pf_output<true>(a, e, p, valid, x, mbar, s, g);
    }
#pragma unroll
    for (int d = 0; d < MAXD; ++d) {
        double v = g[d];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (valid && (threadIdx.x & 31) == 0 && d < a.D) a.gxt[row * a.D + d] = v;
    }
}

int pf_eval_launch(cudaStream_t st, const PfDev& a) {
    launch_hi(pf_eval_kernel, dim3((unsigned)((a.T + PF_WARPS - 1) / PF_WARPS), a.E), dim3(PF_WARPS * 32), 0, st, a);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int pf_vjp_launch(cudaStream_t st, const PfDev& a) {
    launch_hi(pf_vjp_kernel, dim3((unsigned)((a.T + PF_WARPS - 1) / PF_WARPS)), dim3(PF_WARPS * 32), 0, st, a);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

// ---- the draw ----------------------------------------------------------------------------------------------------------
// omega [E,F,D] = zeta / ell_e
__global__ void __launch_bounds__(256) pf_omega_kernel(int E, int F, int D, const double* zeta, const double* ell,
                                                       double* omega) {
    PDL_ENTRY();
    const size_t q = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (q >= (size_t)E * F * D) return;
    const int d = (int)(q % D), e = (int)(q / ((size_t)F * D));
    omega[q] = zeta[q] / ell[(size_t)e * D + d];
}

// Phi_e(X) [E,n,2F]: row j = sqrt(sf2_e / F) [cos(omega_e X_j); sin(omega_e X_j)], grid (ceil(n F / 256), E)
__global__ void __launch_bounds__(256) pf_phi_kernel(int n, int F, int D, const double* X, const double* sf2,
                                                     const double* omega, double* Phi) {
    PDL_ENTRY();
    const size_t q = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (q >= (size_t)n * F) return;
    const int e = blockIdx.y, j = (int)(q / F), i = (int)(q % F);
    const double* om = omega + ((size_t)e * F + i) * D;
    double arg = 0.0;
    for (int d = 0; d < D; ++d) arg = fma(om[d], X[(size_t)j * D + d], arg);
    double sn, cs;
    sincospi(arg * PT_INV_PI, &sn, &cs);
    const double sc = sqrt(sf2[e] / F);
    double* row = Phi + ((size_t)e * n + j) * 2 * F;
    row[i] = sc * cs;
    row[F + i] = sc * sn;
}

// [P,E,n]: R += sqrt(sn2_e) eps, v = beta_e
__global__ void __launch_bounds__(256) pf_prep_kernel(size_t total, int E, int n, const double* sn2, const double* eps,
                                                      const double* beta, double* Rt, double* v) {
    PDL_ENTRY();
    const size_t q = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (q >= total) return;
    const int j = (int)(q % n), e = (int)((q / n) % E);
    Rt[q] = fma(sqrt(sn2[e]), eps[q], Rt[q]);
    v[q] = beta[(size_t)e * n + j];
}

// the draw's workspace: Phi [E,n,2F] and R [P,E,n] doubles; 0 for sizes out of range or on size_t overflow
static size_t pf_draw_bytes(const pilco_gp_model* dyn, int P, int F) {
    if (!dyn || P < 1 || P > PT_MAX_P || F < 1 || F > PILCO_MAX_FEATURES || dyn->n < 1 || dyn->D < 1 ||
        dyn->D > MAXD || dyn->E < 1 || dyn->E > MAXE)
        return 0;
    const size_t E = dyn->E, n = dyn->n;
    size_t phi = 0, r = 0, tot = 0;
    if (__builtin_mul_overflow(E * n, (size_t)2 * F, &phi) || __builtin_mul_overflow((size_t)P * E, n, &r) ||
        __builtin_add_overflow(phi + (phi & 1), r, &tot) || __builtin_mul_overflow(tot, sizeof(double), &tot))
        return 0;
    return tot;
}

extern "C" {

size_t pilco_particles_features_draw_workspace_bytes(const pilco_gp_model* dyn, int P, int F) {
    return pf_draw_bytes(dyn, P, F);
}

int pilco_particles_features_draw(const pilco_gp_model* dyn, const double* sn2, int P, int F, const double* zeta,
                                  const double* w, const double* eps_y, double* omega, double* v, void* ws,
                                  size_t ws_bytes, pilco_stream_t stream) {
    if (!dyn || !sn2 || !zeta || !w || !eps_y || !omega || !v) return PILCO_ERR_NULL;
    if (!dyn->X || !dyn->ell || !dyn->sf2 || !dyn->beta) return PILCO_ERR_NULL;
    if (dyn->mode != 0 || !dyn->iK || dyn->X_bs || dyn->ell_bs || dyn->sf2_bs || dyn->beta_bs)
        return PILCO_ERR_UNSUPPORTED;
    if (dyn->n < 1 || dyn->D < 1 || dyn->D > MAXD || dyn->E < 1 || dyn->E > MAXE || dyn->ldk < pad64(dyn->n) ||
        P < 1 || P > PT_MAX_P || F < 1 || F > PILCO_MAX_FEATURES)
        return PILCO_ERR_DIM;
    const size_t need = pf_draw_bytes(dyn, P, F);
    if (!ws) return PILCO_ERR_NULL;
    if ((uintptr_t)ws & 15) return PILCO_ERR_ALIGN;
    if (need == 0) return PILCO_ERR_DIM;
    if (ws_bytes < need) return PILCO_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    const int E = dyn->E, n = dyn->n, D = dyn->D, F2 = 2 * F;
    const size_t nphi = (size_t)E * n * F2, nr = (size_t)P * E * n;
    double* Phi = (double*)ws;
    double* Rt = Phi + nphi + (nphi & 1);
    const size_t no = (size_t)E * F * D;
    launch_hi(pf_omega_kernel, dim3((unsigned)((no + 255) / 256)), dim3(256), 0, st, E, F, D, zeta, dyn->ell, omega);
    CUDA_LAUNCH_CHECK();
    launch_hi(pf_phi_kernel, dim3((unsigned)(((size_t)n * F + 255) / 256), E), dim3(256), 0, st, n, F, D, dyn->X,
              dyn->sf2, (const double*)omega, Phi);
    CUDA_LAUNCH_CHECK();
    // R_e' [P,n] = W_e' Phi_e(X)': a particle's row is one fixed k-order dot product per column, whatever P
    if (const int rc = gemm(st, E, P, n, F2, 0, 1, 1.0, w, E * F2, F2, Phi, F2, (long long)n * F2, 0.0, Rt, E * n, n))
        return rc;
    launch_hi(pf_prep_kernel, dim3((unsigned)((nr + 255) / 256)), dim3(256), 0, st, nr, E, n, sn2, eps_y, dyn->beta,
              Rt, v);
    CUDA_LAUNCH_CHECK();
    // V_e' = beta_e' - R_e' iK_e (iK symmetric)
    return gemm(st, E, P, n, n, 0, 0, -1.0, Rt, E * n, n, dyn->iK, dyn->ldk, (long long)dyn->ldk * dyn->ldk, 1.0, v,
                E * n, n);
}

}  // extern "C"
