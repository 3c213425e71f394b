// predict.cu -- posterior of the factorised dynamics GPs at T deterministic inputs (fp64):
//   pilco_gp_predict   gpflow GPR.predict_f / GPRFITC.predict_f over the device factors (iK, beta) of
//                      pilco_gp_factorize / pilco_gp_append / pilco_fitc_factorize
//   mean(x) = k*(x)' beta_e,   var(x) = sf2_e - k*(x)' iK_e k*(x),   k*(x)_i = sf2_e exp(-0.5 |(x - c_i)/ell_e|^2)
// The diagonal path is one fused kernel (gp_predict_kernel, DESIGN.md section 10): the quadratic form runs on
// DMMA.16x8x16 with iK tiles staged by TMA bulk copies, K* is computed in shared memory chunk by chunk and never
// written to global memory.  The full covariance is composed from the factorisation building blocks (factorize.cu).
#include "common.cuh"

#define PR_TR   32              // test points per CTA (two m16 row tiles)
#define PR_JB   256             // iK columns per CTA (four warps of 64 columns)
#define PR_KC   16              // iK rows per pipeline stage (one m16n8k16 k-step)
#define PR_LDA  (PR_KC + 4)     // K* chunk row stride: == 4 (mod 16), the A-fragment reads are bank-conflict free
#define PR_LDB  (PR_JB + 4)     // iK tile row stride:  == 4 (mod 16), the B-fragment reads are bank-conflict free

struct PredictArgs {
    int n, D, np, nj, nrb, T, e0;
    const double* C;            // [n,D] centres
    const double* ell;          // [E,D]
    const double* sf2;          // [E]
    const double* beta;         // [E,n]
    const double* iK; int ldk;  // [E,ldk,ldk]
    const double* Xs;           // [T,D]
    double* mean; double* var;  // [T,ne]
    int ne;
    double* part;               // [ne, nrb, nj, 2, PR_TR] partial (quadratic form, mean) sums per j block
    unsigned* cnt;              // [ne, nrb] arrival counters (zeroed by the launcher)
};

struct PredictSmem {
    double B[2][PR_KC * PR_LDB];        // iK[i chunk, j block], double buffered (TMA destination)
    double A[2][PR_TR * PR_LDA];        // K*[rows, i chunk], double buffered
    double x[PR_TR * MAXD];             // test inputs of the CTA's rows
    double il[MAXD];                    // 1 / ell_e
    double red[4][2][PR_TR];            // per column warp: row sums (quadratic form, mean)
    uint64_t bar[2];
};

// k*(x_r)_i: direct difference form (no expanded |x|^2 + |c|^2 - 2 x.c: nothing here centres the inputs)
__device__ __forceinline__ double pr_kstar(const double* x, const double* c, const double* il, int D, double sf2) {
    double d2 = 0.0;
    for (int d = 0; d < D; ++d) { const double t = (x[d] - c[d]) * il[d]; d2 = fma(t, t, d2); }
    return sf2 * exp(-0.5 * d2);
}

// grid (nj, nrb, ne), 256 threads = 8 warps as 2 (row tiles of 16) x 4 (column ranges of 64)
__global__ void __launch_bounds__(256, 2) gp_predict_kernel(PredictArgs a) {
    PDL_ENTRY();
    extern __shared__ __align__(16) unsigned char pr_smem_raw[];
    PredictSmem& sm = *reinterpret_cast<PredictSmem*>(pr_smem_raw);
    const int jb = blockIdx.x, rb = blockIdx.y, z = blockIdx.z, e = a.e0 + z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = (warp >> 2) * 16, wc = warp & 3, wn = wc * 64;
    const int D = a.D, r0 = rb * PR_TR, j0 = jb * PR_JB;
    const int jw = min(PR_JB, a.np - j0);                       // multiple of 64
    const bool active = wn < jw;                                // this warp's 64 columns exist
    const double sf2 = a.sf2[e];
    const double* iK = a.iK + (size_t)e * a.ldk * a.ldk;
    for (int i = tid; i < PR_TR * MAXD; i += 256) {
        const int r = i / MAXD, d = i % MAXD;
        sm.x[i] = (r0 + r < a.T && d < D) ? a.Xs[(size_t)(r0 + r) * D + d] : 0.0;
    }
    if (tid < MAXD) sm.il[tid] = tid < D ? 1.0 / a.ell[(size_t)e * D + tid] : 0.0;
    if (tid == 0) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); mbar_fence_init(); }
    __syncthreads();
    const int nc = a.np / PR_KC;
    auto issue = [&](int c) {                                   // thread 0: iK rows [c KC, (c+1) KC) x [j0, j0 + jw)
        uint64_t* bar = &sm.bar[c & 1];
        mbar_expect_tx(bar, (unsigned)(PR_KC * jw * sizeof(double)));
        for (int k = 0; k < PR_KC; ++k)
            tma_bulk_g2s(&sm.B[c & 1][k * PR_LDB], iK + (size_t)(c * PR_KC + k) * a.ldk + j0, (unsigned)(jw * sizeof(double)), bar);
    };
    auto kchunk = [&](int c) {                                  // K*[rows, c KC .. (c+1) KC) -> A[c & 1]; 0 past n or T
        double* A = sm.A[c & 1];
        for (int q = tid; q < PR_TR * PR_KC; q += 256) {
            const int r = q / PR_KC, k = q % PR_KC, i = c * PR_KC + k;
            double v = 0.0;
            if (i < a.n && r0 + r < a.T) v = pr_kstar(&sm.x[r * MAXD], a.C + (size_t)i * D, sm.il, D, sf2);
            A[r * PR_LDA + k] = v;
        }
    };
    if (tid == 0) { issue(0); if (nc > 1) issue(1); }
    kchunk(0);
    double acc[8][4];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.0;
    for (int c = 0; c < nc; ++c) {
        __syncthreads();                                        // A[c & 1] written; stage (c + 1) & 1 consumed at c - 1
        if (tid == 0 && c >= 1 && c + 1 < nc) issue(c + 1);
        if (c + 1 < nc) kchunk(c + 1);
        mbar_wait(&sm.bar[c & 1], (unsigned)((c >> 1) & 1));
        if (active) {
            const double* A = sm.A[c & 1];
            const double* B = sm.B[c & 1];
            double af[8];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                af[2 * i] = A[(wm + g) * PR_LDA + t + 4 * i];
                af[2 * i + 1] = A[(wm + g + 8) * PR_LDA + t + 4 * i];
            }
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                double bf[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) bf[i] = B[(t + 4 * i) * PR_LDB + wn + 8 * q + g];
                dmma16816(acc[q], af, bf);
            }
        }
    }
    // epilogue: W = K* iK[:, j block] is in acc (rows wm + g, wm + g + 8; columns wn + 8q + 2t + {0,1}).  Row dot with
    // K*[rows, j block] (recomputed: same function, same bits) and the mean partial K*[rows, j block] beta[j block].
    double qf[2] = {0.0, 0.0}, mp[2] = {0.0, 0.0};
    if (active) {
        const double* be = a.beta + (size_t)e * a.n;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = wm + g + 8 * h;
            if (r0 + r < a.T) {
#pragma unroll
                for (int q = 0; q < 8; ++q)
#pragma unroll
                    for (int o = 0; o < 2; ++o) {
                        const int j = j0 + wn + 8 * q + 2 * t + o;
                        if (j < a.n) {
                            const double k = pr_kstar(&sm.x[r * MAXD], a.C + (size_t)j * D, sm.il, D, sf2);
                            qf[h] = fma(acc[q][2 * h + o], k, qf[h]);
                            mp[h] = fma(k, be[j], mp[h]);
                        }
                    }
            }
        }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {                               // over the four t lanes of a row: fixed butterfly
        qf[h] += __shfl_xor_sync(0xffffffffu, qf[h], 1);
        qf[h] += __shfl_xor_sync(0xffffffffu, qf[h], 2);
        mp[h] += __shfl_xor_sync(0xffffffffu, mp[h], 1);
        mp[h] += __shfl_xor_sync(0xffffffffu, mp[h], 2);
    }
    if (t == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) { sm.red[wc][0][wm + g + 8 * h] = qf[h]; sm.red[wc][1][wm + g + 8 * h] = mp[h]; }
    }
    __syncthreads();
    double* part = a.part + (((size_t)z * a.nrb + rb) * a.nj) * 2 * PR_TR;
    if (tid < 2 * PR_TR) {                                      // column warps in fixed order
        const int w = tid / PR_TR, r = tid % PR_TR;
        part[(size_t)jb * 2 * PR_TR + tid] = ((sm.red[0][w][r] + sm.red[1][w][r]) + sm.red[2][w][r]) + sm.red[3][w][r];
    }
    if (!last_cta_arrives(a.cnt + (size_t)z * a.nrb + rb, (unsigned)a.nj)) return;
    if (tid < PR_TR && r0 + tid < a.T) {                        // j blocks in fixed order
        double qs = 0.0, ms = 0.0;
        for (int b = 0; b < a.nj; ++b) { qs += part[(size_t)b * 2 * PR_TR + tid]; ms += part[(size_t)b * 2 * PR_TR + PR_TR + tid]; }
        a.mean[(size_t)(r0 + tid) * a.ne + z] = ms;
        a.var[(size_t)(r0 + tid) * a.ne + z] = sf2 - qs;
    }
}

// ---- VJP of the diagonal posterior at the inputs (pilco_gp_predict_vjp, DESIGN.md section 12) ----------------------
//   gx = sum_e ell_e^-2 o sum_n c_en (c_n - x),   c_en = k_en (gmean_e beta_en - 2 gvar_e w_en),   w_e = iK_e k_e
// (d k_en / dx = k_en (c_n - x) / ell_e^2; d var / d k = -2 w since iK is symmetric).  The difference form c_n - x is
// summed directly: the expanded sum_n c_n c_n - (sum_n c_n) x would cancel when |x| >> |c_n - x|.
struct VjpArgs {
    int n, D, np, nj, nrb, T, E;
    const double* C; const double* ell; const double* sf2; const double* beta;
    const double* iK; int ldk;
    const double* Xs;           // [T,D]
    const double* gmean;        // [T,E]
    const double* gvar;         // [T,E]
    double* gXs;                // [T,D]
    double* part;               // [E, nrb, nj, PR_TR, D] per-(output, j block) sums of c_en (c_n - x)
    unsigned* cnt;              // [nrb] arrival counters over the nj * E CTAs of a row block (zeroed by the launcher)
};

struct VjpSmem {
    double B[2][PR_KC * PR_LDB];        // iK[i chunk, j block] (TMA destination); after the main loop c [PR_TR][PR_LDB]
    double A[2][PR_TR * PR_LDA];        // K*[rows, i chunk]
    double x[PR_TR * MAXD];
    double il[MAXD];
    double gm[PR_TR], gv[PR_TR];        // the rows' cotangents of output e
    uint64_t bar[2];
};
static_assert(2 * PR_KC >= PR_TR, "c of the CTA's rows x j block fits the iK double buffer");

// grid (nj, nrb, E), 256 threads.  The main loop is gp_predict_kernel's (W = K* iK[:, j block] on DMMA.16x8x16 from
// TMA-staged iK tiles); only the epilogue differs: c for the CTA's (rows, j block) goes to the free iK buffer, then
// 8 lanes per row sum c (c_n - x) over the block's columns in a fixed order and the last of the row block's nj * E
// CTAs applies ell_e^-2 and sums the outputs and j blocks in a fixed order.
__global__ void __launch_bounds__(256, 2) gp_predict_vjp_kernel(VjpArgs a) {
    PDL_ENTRY();
    extern __shared__ __align__(16) unsigned char pr_smem_raw[];
    VjpSmem& sm = *reinterpret_cast<VjpSmem*>(pr_smem_raw);
    const int jb = blockIdx.x, rb = blockIdx.y, e = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = (warp >> 2) * 16, wc = warp & 3, wn = wc * 64;
    const int D = a.D, r0 = rb * PR_TR, j0 = jb * PR_JB;
    const int jw = min(PR_JB, a.np - j0);
    const bool active = wn < jw;
    const double sf2 = a.sf2[e];
    const double* iK = a.iK + (size_t)e * a.ldk * a.ldk;
    for (int i = tid; i < PR_TR * MAXD; i += 256) {
        const int r = i / MAXD, d = i % MAXD;
        sm.x[i] = (r0 + r < a.T && d < D) ? a.Xs[(size_t)(r0 + r) * D + d] : 0.0;
    }
    if (tid < MAXD) sm.il[tid] = tid < D ? 1.0 / a.ell[(size_t)e * D + tid] : 0.0;
    if (tid < PR_TR) {
        const bool in = r0 + tid < a.T;
        sm.gm[tid] = in ? a.gmean[(size_t)(r0 + tid) * a.E + e] : 0.0;
        sm.gv[tid] = in ? a.gvar[(size_t)(r0 + tid) * a.E + e] : 0.0;
    }
    if (tid == 0) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); mbar_fence_init(); }
    __syncthreads();
    // main loop: gp_predict_kernel's, kept as its own copy so that the predict kernel's code is not touched
    const int nc = a.np / PR_KC;
    auto issue = [&](int c) {
        uint64_t* bar = &sm.bar[c & 1];
        mbar_expect_tx(bar, (unsigned)(PR_KC * jw * sizeof(double)));
        for (int k = 0; k < PR_KC; ++k)
            tma_bulk_g2s(&sm.B[c & 1][k * PR_LDB], iK + (size_t)(c * PR_KC + k) * a.ldk + j0, (unsigned)(jw * sizeof(double)), bar);
    };
    auto kchunk = [&](int c) {
        double* A = sm.A[c & 1];
        for (int q = tid; q < PR_TR * PR_KC; q += 256) {
            const int r = q / PR_KC, k = q % PR_KC, i = c * PR_KC + k;
            double v = 0.0;
            if (i < a.n && r0 + r < a.T) v = pr_kstar(&sm.x[r * MAXD], a.C + (size_t)i * D, sm.il, D, sf2);
            A[r * PR_LDA + k] = v;
        }
    };
    if (tid == 0) { issue(0); if (nc > 1) issue(1); }
    kchunk(0);
    double acc[8][4];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.0;
    for (int c = 0; c < nc; ++c) {
        __syncthreads();
        if (tid == 0 && c >= 1 && c + 1 < nc) issue(c + 1);
        if (c + 1 < nc) kchunk(c + 1);
        mbar_wait(&sm.bar[c & 1], (unsigned)((c >> 1) & 1));
        if (active) {
            const double* A = sm.A[c & 1];
            const double* B = sm.B[c & 1];
            double af[8];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                af[2 * i] = A[(wm + g) * PR_LDA + t + 4 * i];
                af[2 * i + 1] = A[(wm + g + 8) * PR_LDA + t + 4 * i];
            }
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                double bf[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) bf[i] = B[(t + 4 * i) * PR_LDB + wn + 8 * q + g];
                dmma16816(acc[q], af, bf);
            }
        }
    }
    __syncthreads();                                            // every warp is done with the last iK tile
    double* cs = &sm.B[0][0];                                   // c [PR_TR][PR_LDB]
    const double* be = a.beta + (size_t)e * a.n;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = wm + g + 8 * h;
#pragma unroll
        for (int q = 0; q < 8; ++q)
#pragma unroll
            for (int o = 0; o < 2; ++o) {
                const int jl = wn + 8 * q + 2 * t + o, j = j0 + jl;
                double c = 0.0;
                if (active && r0 + r < a.T && j < a.n) {
                    const double k = pr_kstar(&sm.x[r * MAXD], a.C + (size_t)j * D, sm.il, D, sf2);
                    c = k * fma(-2.0 * sm.gv[r], acc[q][2 * h + o], sm.gm[r] * be[j]);
                }
                cs[r * PR_LDB + jl] = c;
            }
    }
    __syncthreads();
    {                                                           // row r = tid / 8; lane s sums columns s, s + 8, ...
        const int r = tid >> 3, s = tid & 7;
        const int jend = min(PR_JB, a.n - j0);
        const double* xr = &sm.x[r * MAXD];
        double gs[MAXD];
#pragma unroll
        for (int d = 0; d < MAXD; ++d) gs[d] = 0.0;
        for (int jl = s; jl < jend; jl += 8) {
            const double c = cs[r * PR_LDB + jl];
            const double* cj = a.C + (size_t)(j0 + jl) * D;
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < D) gs[d] = fma(c, cj[d] - xr[d], gs[d]);
        }
#pragma unroll
        for (int d = 0; d < MAXD; ++d) {                        // over the 8 lanes of a row: fixed butterfly
            gs[d] += __shfl_xor_sync(0xffffffffu, gs[d], 1);
            gs[d] += __shfl_xor_sync(0xffffffffu, gs[d], 2);
            gs[d] += __shfl_xor_sync(0xffffffffu, gs[d], 4);
        }
        if (s == 0 && r0 + r < a.T) {
            double* pr = a.part + ((((size_t)e * a.nrb + rb) * a.nj + jb) * PR_TR + r) * D;
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < D) pr[d] = gs[d];
        }
    }
    if (!last_cta_arrives(a.cnt + rb, (unsigned)(a.nj * a.E))) return;
    for (int q = tid; q < PR_TR * D; q += 256) {                // outputs, then j blocks, in fixed order
        const int r = q / D, d = q % D;
        if (r0 + r >= a.T) continue;
        double sum = 0.0;
        for (int ee = 0; ee < a.E; ++ee) {
            const double* pe = a.part + (((size_t)ee * a.nrb + rb) * a.nj * PR_TR + r) * D + d;
            double se = 0.0;
            for (int b = 0; b < a.nj; ++b) se += pe[(size_t)b * PR_TR * D];
            const double il = 1.0 / a.ell[(size_t)ee * D + d];
            sum = fma(se, il * il, sum);
        }
        a.gXs[(size_t)(r0 + r) * D + d] = sum;
    }
}

// ---- predict for the consistent particle sampler (pilco_particles_rollout_consistent, DESIGN.md section 14) ---------
// gp_predict_kernel with two extra epilogue stores of values it already holds: W = K* iK (the C fragments) to
// W[e, row, :] and the recomputed K* to Ks[e, row, :], both [ne, T, np] with zeros past n.  mean and var are bitwise
// those of pilco_gp_predict at the same inputs (same main loop, same epilogue order, same reductions).
struct FsPredArgs {
    PredictArgs p;
    double* W;                  // [ne, T, np]  K* iK
    double* Ks;                 // [ne, T, np]  K*
};

// grid (nj, nrb, ne), 256 threads: gp_predict_kernel's decomposition
__global__ void __launch_bounds__(256, 2) fs_predict_kernel(FsPredArgs fa) {
    PDL_ENTRY();
    const PredictArgs& a = fa.p;
    extern __shared__ __align__(16) unsigned char pr_smem_raw[];
    PredictSmem& sm = *reinterpret_cast<PredictSmem*>(pr_smem_raw);
    const int jb = blockIdx.x, rb = blockIdx.y, z = blockIdx.z, e = a.e0 + z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = (warp >> 2) * 16, wc = warp & 3, wn = wc * 64;
    const int D = a.D, r0 = rb * PR_TR, j0 = jb * PR_JB;
    const int jw = min(PR_JB, a.np - j0);
    const bool active = wn < jw;
    const double sf2 = a.sf2[e];
    const double* iK = a.iK + (size_t)e * a.ldk * a.ldk;
    for (int i = tid; i < PR_TR * MAXD; i += 256) {
        const int r = i / MAXD, d = i % MAXD;
        sm.x[i] = (r0 + r < a.T && d < D) ? a.Xs[(size_t)(r0 + r) * D + d] : 0.0;
    }
    if (tid < MAXD) sm.il[tid] = tid < D ? 1.0 / a.ell[(size_t)e * D + tid] : 0.0;
    if (tid == 0) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); mbar_fence_init(); }
    __syncthreads();
    // main loop: gp_predict_kernel's, kept as its own copy so that the predict kernel's code is not touched
    const int nc = a.np / PR_KC;
    auto issue = [&](int c) {
        uint64_t* bar = &sm.bar[c & 1];
        mbar_expect_tx(bar, (unsigned)(PR_KC * jw * sizeof(double)));
        for (int k = 0; k < PR_KC; ++k)
            tma_bulk_g2s(&sm.B[c & 1][k * PR_LDB], iK + (size_t)(c * PR_KC + k) * a.ldk + j0, (unsigned)(jw * sizeof(double)), bar);
    };
    auto kchunk = [&](int c) {
        double* A = sm.A[c & 1];
        for (int q = tid; q < PR_TR * PR_KC; q += 256) {
            const int r = q / PR_KC, k = q % PR_KC, i = c * PR_KC + k;
            double v = 0.0;
            if (i < a.n && r0 + r < a.T) v = pr_kstar(&sm.x[r * MAXD], a.C + (size_t)i * D, sm.il, D, sf2);
            A[r * PR_LDA + k] = v;
        }
    };
    if (tid == 0) { issue(0); if (nc > 1) issue(1); }
    kchunk(0);
    double acc[8][4];
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.0;
    for (int c = 0; c < nc; ++c) {
        __syncthreads();
        if (tid == 0 && c >= 1 && c + 1 < nc) issue(c + 1);
        if (c + 1 < nc) kchunk(c + 1);
        mbar_wait(&sm.bar[c & 1], (unsigned)((c >> 1) & 1));
        if (active) {
            const double* A = sm.A[c & 1];
            const double* B = sm.B[c & 1];
            double af[8];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                af[2 * i] = A[(wm + g) * PR_LDA + t + 4 * i];
                af[2 * i + 1] = A[(wm + g + 8) * PR_LDA + t + 4 * i];
            }
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                double bf[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) bf[i] = B[(t + 4 * i) * PR_LDB + wn + 8 * q + g];
                dmma16816(acc[q], af, bf);
            }
        }
    }
    // epilogue.  W (0 past n) goes to the free iK buffer and out to global memory as coalesced 16-byte rows; then
    // gp_predict_kernel's sums in its order, with each thread's W entries read back from the buffer (the same values)
    // and overwritten by K*, which goes out the same way.
    __syncthreads();                                            // every warp is done with the last iK tile
    double* cs = &sm.B[0][0];                                   // [PR_TR][PR_LDB]
    const int jw2 = jw >> 1;
    auto store_tile = [&](double* dst) {                        // cs rows < T, columns [0, jw) -> dst[z, r0 + r, j0 ..]
        for (int i = tid; i < PR_TR * jw2; i += 256) {
            const int r = i / jw2, c2 = i % jw2;
            if (r0 + r < a.T)
                *reinterpret_cast<double2*>(dst + ((size_t)z * a.T + r0 + r) * a.np + j0 + 2 * c2) =
                    *reinterpret_cast<const double2*>(cs + r * PR_LDB + 2 * c2);
        }
    };
    if (active) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int q = 0; q < 8; ++q)
#pragma unroll
                for (int o = 0; o < 2; ++o) {
                    const int jl = wn + 8 * q + 2 * t + o;
                    cs[(wm + g + 8 * h) * PR_LDB + jl] = j0 + jl < a.n ? acc[q][2 * h + o] : 0.0;
                }
    }
    __syncthreads();
    store_tile(fa.W);
    __syncthreads();                                            // W is out before K* overwrites it
    double qf[2] = {0.0, 0.0}, mp[2] = {0.0, 0.0};
    if (active) {
        const double* be = a.beta + (size_t)e * a.n;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = wm + g + 8 * h;
            if (r0 + r < a.T) {
                for (int q = 0; q < 8; ++q)
#pragma unroll
                    for (int o = 0; o < 2; ++o) {
                        const int j = j0 + wn + 8 * q + 2 * t + o;
                        double* c = &cs[r * PR_LDB + wn + 8 * q + 2 * t + o];
                        double k = 0.0;
                        if (j < a.n) {
                            k = pr_kstar(&sm.x[r * MAXD], a.C + (size_t)j * D, sm.il, D, sf2);
                            qf[h] = fma(*c, k, qf[h]);
                            mp[h] = fma(k, be[j], mp[h]);
                        }
                        *c = k;
                    }
            }
        }
    }
    __syncthreads();
    store_tile(fa.Ks);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        qf[h] += __shfl_xor_sync(0xffffffffu, qf[h], 1);
        qf[h] += __shfl_xor_sync(0xffffffffu, qf[h], 2);
        mp[h] += __shfl_xor_sync(0xffffffffu, mp[h], 1);
        mp[h] += __shfl_xor_sync(0xffffffffu, mp[h], 2);
    }
    if (t == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) { sm.red[wc][0][wm + g + 8 * h] = qf[h]; sm.red[wc][1][wm + g + 8 * h] = mp[h]; }
    }
    __syncthreads();
    double* part = a.part + (((size_t)z * a.nrb + rb) * a.nj) * 2 * PR_TR;
    if (tid < 2 * PR_TR) {
        const int w = tid / PR_TR, r = tid % PR_TR;
        part[(size_t)jb * 2 * PR_TR + tid] = ((sm.red[0][w][r] + sm.red[1][w][r]) + sm.red[2][w][r]) + sm.red[3][w][r];
    }
    if (!last_cta_arrives(a.cnt + (size_t)z * a.nrb + rb, (unsigned)a.nj)) return;
    if (tid < PR_TR && r0 + tid < a.T) {
        double qs = 0.0, ms = 0.0;
        for (int b = 0; b < a.nj; ++b) { qs += part[(size_t)b * 2 * PR_TR + tid]; ms += part[(size_t)b * 2 * PR_TR + PR_TR + tid]; }
        a.mean[(size_t)(r0 + tid) * a.ne + z] = ms;
        a.var[(size_t)(r0 + tid) * a.ne + z] = sf2 - qs;
    }
}

// one-time kernel attribute of fs_predict_kernel (before the consistent rollout enqueues anything)
int fs_predict_prepare() {
    static bool attr_set[PILCO_MAX_DEVICES] = {false};
    bool& set = attr_set[pilco_current_device()];
    if (!set) {
        if (cudaFuncSetAttribute(fs_predict_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PredictSmem))
            != cudaSuccess)
            return PILCO_ERR_LAUNCH;
        set = true;
    }
    return PILCO_OK;
}

// all ne = E outputs of the validated model at T points (T <= 65535 * PR_TR); ws: pilco_gp_predict's diagonal workspace
int fs_predict_launch(cudaStream_t st, const pilco_gp_model* gp, int T, const double* Xs, double* mean, double* var,
                      double* W, double* Ks, void* ws) {
    const int n = gp->n, E = gp->E, np = pad64(n), nj = (np + PR_JB - 1) / PR_JB, nrb = (T + PR_TR - 1) / PR_TR;
    FsPredArgs fa;
    PredictArgs& a = fa.p;
    a.n = n; a.D = gp->D; a.np = np; a.nj = nj; a.nrb = nrb; a.T = T; a.e0 = 0;
    a.C = gp->X; a.ell = gp->ell; a.sf2 = gp->sf2; a.beta = gp->beta; a.iK = gp->iK; a.ldk = gp->ldk;
    a.Xs = Xs; a.mean = mean; a.var = var; a.ne = E;
    a.part = (double*)ws;
    a.cnt = (unsigned*)((char*)ws + (size_t)E * nrb * nj * 2 * PR_TR * sizeof(double));
    fa.W = W; fa.Ks = Ks;
    cudaMemsetAsync(a.cnt, 0, (size_t)E * nrb * sizeof(unsigned), st);
    const dim3 grid(nj, nrb, E);
    launch_pri(pilco_small_grid(grid), fs_predict_kernel, grid, dim3(256), sizeof(PredictSmem), st, fa);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

static size_t pr_vjp_bytes(int np, int D, int E, int T) {
    const size_t nj = (size_t)(np + PR_JB - 1) / PR_JB, nrb = (size_t)(T + PR_TR - 1) / PR_TR;
    const size_t part = (size_t)E * nrb * nj * PR_TR * D * sizeof(double);
    const size_t cnt = (nrb * sizeof(unsigned) + 15) & ~(size_t)15;
    return part + cnt;
}

// full covariance (factorize.cu): K*, K** (gram_kernel), W = K* iK, K** - W K*' and K* beta (gemm)
int gp_predict_full_cov(cudaStream_t st, int n, int D, int ne, int T, const double* C, const double* ell, const double* sf2,
                        const double* beta, const double* iK, int ldk, const double* Xs, double* mean, double* cov, double* ws);

static size_t pr_diag_bytes(int np, int ne, int T) {
    const size_t nj = (size_t)(np + PR_JB - 1) / PR_JB, nrb = (size_t)(T + PR_TR - 1) / PR_TR;
    const size_t part = (size_t)ne * nrb * nj * 2 * PR_TR * sizeof(double);
    const size_t cnt = ((size_t)ne * nrb * sizeof(unsigned) + 15) & ~(size_t)15;
    return part + cnt;
}

extern "C" {

size_t pilco_gp_predict_workspace_bytes(int n, int D, int E, int T, int full_cov) {
    if (n < 1 || D < 1 || D > MAXD || E < 1 || E > MAXE || T < 1 || T > 65535 * PR_TR) return 0;
    const int np = pad64(n);
    if (full_cov) return T > 65535 * 8 ? 0 : 2 * (size_t)E * T * np * sizeof(double);    // K*, W = K* iK  [E,T,np] each
    return pr_diag_bytes(np, E, T);
}

int pilco_gp_predict(const pilco_gp_model* gp, int e0, int ne, int T, const double* Xs, double* mean, double* var,
                     int full_cov, void* ws, size_t ws_bytes, pilco_stream_t stream) {
    if (!gp || !Xs || !mean || !var || !ws) return PILCO_ERR_NULL;
    if (!gp->X || !gp->ell || !gp->sf2 || !gp->beta) return PILCO_ERR_NULL;
    if (gp->mode != 0 || !gp->iK || gp->X_bs || gp->ell_bs || gp->sf2_bs || gp->beta_bs) return PILCO_ERR_UNSUPPORTED;
    const int n = gp->n, D = gp->D, E = gp->E;
    if (n < 1 || D < 1 || D > MAXD || E < 1 || E > MAXE) return PILCO_ERR_DIM;
    if (T < 1 || T > (full_cov ? 65535 * 8 : 65535 * PR_TR) || ne < 1 || e0 < 0 || e0 + ne > E) return PILCO_ERR_DIM;
    if (gp->ldk < pad64(n)) return PILCO_ERR_DIM;
    if (((uintptr_t)gp->iK & 15) || (gp->ldk & 1) || ((uintptr_t)ws & 15)) return PILCO_ERR_ALIGN;   // TMA rows: 16 B
    if (ws_bytes < pilco_gp_predict_workspace_bytes(n, D, ne, T, full_cov)) return PILCO_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    if (full_cov)
        return gp_predict_full_cov(st, n, D, ne, T, gp->X, gp->ell + (size_t)e0 * D, gp->sf2 + e0, gp->beta + (size_t)e0 * n,
                                   gp->iK + (size_t)e0 * gp->ldk * gp->ldk, gp->ldk, Xs, mean, var, (double*)ws);
    const int np = pad64(n), nj = (np + PR_JB - 1) / PR_JB, nrb = (T + PR_TR - 1) / PR_TR;
    PredictArgs a;
    a.n = n; a.D = D; a.np = np; a.nj = nj; a.nrb = nrb; a.T = T; a.e0 = e0;
    a.C = gp->X; a.ell = gp->ell; a.sf2 = gp->sf2; a.beta = gp->beta; a.iK = gp->iK; a.ldk = gp->ldk;
    a.Xs = Xs; a.mean = mean; a.var = var; a.ne = ne;
    a.part = (double*)ws;
    a.cnt = (unsigned*)((char*)ws + (size_t)ne * nrb * nj * 2 * PR_TR * sizeof(double));
    cudaMemsetAsync(a.cnt, 0, (size_t)ne * nrb * sizeof(unsigned), st);
    const size_t smem = sizeof(PredictSmem);
    static bool attr_set[PILCO_MAX_DEVICES] = {false};
    bool& set = attr_set[pilco_current_device()];
    if (!set) {
        if (cudaFuncSetAttribute(gp_predict_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
            return PILCO_ERR_LAUNCH;
        set = true;
    }
    const dim3 grid(nj, nrb, ne);
    launch_pri(pilco_small_grid(grid), gp_predict_kernel, grid, dim3(256), smem, st, a);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

size_t pilco_gp_predict_vjp_workspace_bytes(int n, int D, int E, int T) {
    if (n < 1 || D < 1 || D > MAXD || E < 1 || E > MAXE || T < 1 || T > 65535 * PR_TR) return 0;
    return pr_vjp_bytes(pad64(n), D, E, T);
}

int pilco_gp_predict_vjp(const pilco_gp_model* gp, int T, const double* Xs, const double* gmean, const double* gvar,
                         double* gXs, void* ws, size_t ws_bytes, pilco_stream_t stream) {
    if (!gp || !Xs || !gmean || !gvar || !gXs || !ws) return PILCO_ERR_NULL;
    if (!gp->X || !gp->ell || !gp->sf2 || !gp->beta) return PILCO_ERR_NULL;
    if (gp->mode != 0 || !gp->iK || gp->X_bs || gp->ell_bs || gp->sf2_bs || gp->beta_bs) return PILCO_ERR_UNSUPPORTED;
    const int n = gp->n, D = gp->D, E = gp->E;
    if (n < 1 || D < 1 || D > MAXD || E < 1 || E > MAXE) return PILCO_ERR_DIM;
    if (T < 1 || T > 65535 * PR_TR) return PILCO_ERR_DIM;
    if (gp->ldk < pad64(n)) return PILCO_ERR_DIM;
    if (((uintptr_t)gp->iK & 15) || (gp->ldk & 1) || ((uintptr_t)ws & 15)) return PILCO_ERR_ALIGN;
    if (ws_bytes < pilco_gp_predict_vjp_workspace_bytes(n, D, E, T)) return PILCO_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    const int np = pad64(n), nj = (np + PR_JB - 1) / PR_JB, nrb = (T + PR_TR - 1) / PR_TR;
    VjpArgs a;
    a.n = n; a.D = D; a.np = np; a.nj = nj; a.nrb = nrb; a.T = T; a.E = E;
    a.C = gp->X; a.ell = gp->ell; a.sf2 = gp->sf2; a.beta = gp->beta; a.iK = gp->iK; a.ldk = gp->ldk;
    a.Xs = Xs; a.gmean = gmean; a.gvar = gvar; a.gXs = gXs;
    a.part = (double*)ws;
    a.cnt = (unsigned*)((char*)ws + (size_t)E * nrb * nj * PR_TR * D * sizeof(double));
    cudaMemsetAsync(a.cnt, 0, (size_t)nrb * sizeof(unsigned), st);
    const size_t smem = sizeof(VjpSmem);
    static bool attr_set[PILCO_MAX_DEVICES] = {false};
    bool& set = attr_set[pilco_current_device()];
    if (!set) {
        if (cudaFuncSetAttribute(gp_predict_vjp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
            return PILCO_ERR_LAUNCH;
        set = true;
    }
    const dim3 grid(nj, nrb, E);
    launch_pri(pilco_small_grid(grid), gp_predict_vjp_kernel, grid, dim3(256), smem, st, a);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

}  // extern "C"
