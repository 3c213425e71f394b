// predict.cu -- posterior of the factorised dynamics GPs at T deterministic inputs (fp64):
//   pilco_gp_predict   gpflow GPR.predict_f / GPRFITC.predict_f over the device factors (iK, beta) of
//                      pilco_gp_factorize / pilco_gp_append_tri / pilco_fitc_factorize
//   mean(x) = k*(x)' beta_e,   var(x) = sf2_e - k*(x)' iK_e k*(x),   k*(x)_i = sf2_e exp(-0.5 |(x - c_i)/ell_e|^2)
// The diagonal path is one fused kernel (gp_predict_kernel, DESIGN.md section 10): the quadratic form runs on
// DMMA.16x8x16 with iK tiles staged by TMA bulk copies, K* is computed in shared memory chunk by chunk and never
// written to global memory.  The full covariance is composed from the factorisation building blocks (factorize.cu).
// The four kernels of the family (the predict and its VJP, and their variants for the consistent particle sampler)
// share the prologue, the main loop (pr_main_loop) and, per family, the reduction tail.
#include "common.cuh"

#define PR_TR   32              // test points per CTA (two m16 row tiles)
#define PR_JB   256             // iK columns per CTA (four warps of 64 columns)
#define PR_KC   16              // iK rows per pipeline stage (one m16n8k16 k-step)
#define PR_LDA  (PR_KC + 4)     // K* chunk row stride: == 4 (mod 16), the A-fragment reads are bank-conflict free
#define PR_LDB  (PR_JB + 4)     // iK tile row stride:  == 4 (mod 16), the B-fragment reads are bank-conflict free

// the model, the points and the grid: what every kernel of the family reads
struct PrArgs {
    int n, D, np, nj, nrb, T;
    const double* C;            // [n,D] centres
    const double* ell;          // [E,D]
    const double* sf2;          // [E]
    const double* beta;         // [E,n]
    const double* iK; int ldk;  // [E,ldk,ldk]
    const double* Xs;           // [T,D]
    double* part;               // per-(row block, j block) partial sums (layout: pr_diag_ws / pr_vjp_ws)
    unsigned* cnt;              // arrival counters (zeroed by the launcher)
};

struct PredictArgs : PrArgs {
    int e0, ne;
    double* mean; double* var;  // [T,ne]
};

// the main loop's shared memory
struct PrTile {
    double B[2][PR_KC * PR_LDB];        // iK[i chunk, j block], double buffered (TMA destination)
    double A[2][PR_TR * PR_LDA];        // A operand [rows, i chunk], double buffered
    double x[PR_TR * MAXD];             // test inputs of the CTA's rows
    double il[MAXD];                    // 1 / ell_e
    uint64_t bar[2];
};

struct PredictSmem {
    PrTile s;
    double red[4][2][PR_TR];            // per column warp: row sums (quadratic form, mean)
};

// k*(x_r)_i: direct difference form (no expanded |x|^2 + |c|^2 - 2 x.c: nothing here centres the inputs)
__device__ __forceinline__ double pr_kstar(const double* x, const double* c, const double* il, int D, double sf2) {
    double d2 = 0.0;
    for (int d = 0; d < D; ++d) { const double t = (x[d] - c[d]) * il[d]; d2 = fma(t, t, d2); }
    return sf2 * exp(-0.5 * d2);
}

// A CTA of grid (nj, nrb, outputs), 256 threads = 8 warps as 2 (row tiles of 16) x 4 (column ranges of 64)
struct PrCta {
    int jb, rb, tid, g, t, wm, wc, wn, r0, j0, jw;
    bool active;                                                // this warp's 64 columns exist
    __device__ __forceinline__ explicit PrCta(int np) {
        jb = blockIdx.x; rb = blockIdx.y; tid = threadIdx.x;
        const int lane = tid & 31, warp = tid >> 5;
        g = lane >> 2; t = lane & 3;
        wm = (warp >> 2) * 16; wc = warp & 3; wn = wc * 64;
        r0 = rb * PR_TR; j0 = jb * PR_JB;
        jw = min(PR_JB, np - j0);                               // multiple of 64
        active = wn < jw;
    }
};

// prologue: the CTA's rows of Xs (0 past T) and 1 / ell_e to shared memory, the two mbarriers initialised
__device__ __forceinline__ void pr_stage(PrTile& sm, const PrCta& q, const PrArgs& a, int e) {
    const int D = a.D;
    for (int i = q.tid; i < PR_TR * MAXD; i += 256) {
        const int r = i / MAXD, d = i % MAXD;
        sm.x[i] = (q.r0 + r < a.T && d < D) ? a.Xs[(size_t)(q.r0 + r) * D + d] : 0.0;
    }
    if (q.tid < MAXD) sm.il[q.tid] = q.tid < D ? 1.0 / a.ell[(size_t)e * D + q.tid] : 0.0;
    if (q.tid == 0) { mbar_init(&sm.bar[0], 1); mbar_init(&sm.bar[1], 1); mbar_fence_init(); }
    __syncthreads();
}

// fill functor of the main loop: K*[rows, c KC .. (c+1) KC) -> A; 0 past n or T.  It captures values, not the
// argument struct: through references the kernels' epilogues unroll less (fewer DFMA/MUFU in the SASS).
__device__ __forceinline__ auto pr_kstar_fill(const PrTile& sm, const PrCta& q, const PrArgs& a, double sf2) {
    const int n = a.n, T = a.T, D = a.D, r0 = q.r0, tid = q.tid;
    const double* C = a.C;
    return [&sm, n, T, D, r0, tid, C, sf2](double* A, int c) {
        for (int k2 = tid; k2 < PR_TR * PR_KC; k2 += 256) {
            const int r = k2 / PR_KC, k = k2 % PR_KC, i = c * PR_KC + k;
            double v = 0.0;
            if (i < n && r0 + r < T) v = pr_kstar(&sm.x[r * MAXD], C + (size_t)i * D, sm.il, D, sf2);
            A[r * PR_LDA + k] = v;
        }
    };
}

// main loop: acc = A iK_e[:, j block] on DMMA.16x8x16 (rows wm + g, wm + g + 8; columns wn + 8q + 2t + {0,1}).
// Thread 0 issues the TMA copies of iK rows [c KC, (c+1) KC) x [j0, j0 + jw) into B[c & 1]; every thread runs
// fill(A[c & 1], c) for the A operand's chunk c one stage ahead.
template <class Fill>
__device__ __forceinline__ void pr_main_loop(PrTile& sm, const PrCta& q, const PrArgs& a, int e, Fill fill,
                                             double (&acc)[8][4]) {
    const double* iK = a.iK + (size_t)e * a.ldk * a.ldk;
    const int nc = a.np / PR_KC;
    auto issue = [&](int c) {
        uint64_t* bar = &sm.bar[c & 1];
        mbar_expect_tx(bar, (unsigned)(PR_KC * q.jw * sizeof(double)));
        for (int k = 0; k < PR_KC; ++k)
            tma_bulk_g2s(&sm.B[c & 1][k * PR_LDB], iK + (size_t)(c * PR_KC + k) * a.ldk + q.j0,
                         (unsigned)(q.jw * sizeof(double)), bar);
    };
    if (q.tid == 0) { issue(0); if (nc > 1) issue(1); }
    fill(sm.A[0], 0);
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k][0] = acc[k][1] = acc[k][2] = acc[k][3] = 0.0;
    for (int c = 0; c < nc; ++c) {
        __syncthreads();                                        // A[c & 1] written; stage (c + 1) & 1 consumed at c - 1
        if (q.tid == 0 && c >= 1 && c + 1 < nc) issue(c + 1);
        if (c + 1 < nc) fill(sm.A[(c + 1) & 1], c + 1);
        mbar_wait(&sm.bar[c & 1], (unsigned)((c >> 1) & 1));
        if (q.active) {
            const double* A = sm.A[c & 1];
            const double* B = sm.B[c & 1];
            double af[8];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                af[2 * i] = A[(q.wm + q.g) * PR_LDA + q.t + 4 * i];
                af[2 * i + 1] = A[(q.wm + q.g + 8) * PR_LDA + q.t + 4 * i];
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                double bf[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) bf[i] = B[(q.t + 4 * i) * PR_LDB + q.wn + 8 * k + q.g];
                dmma16816(acc[k], af, bf);
            }
        }
    }
}

// predict tail: the thread's quadratic form and mean partials qf, mp of rows wm + g + 8h go over the four t lanes of a
// row (fixed butterfly), then the column warps in fixed order to part; the last of the row block's nj CTAs sums the j
// blocks in fixed order into mean and var of output z
__device__ __forceinline__ void pr_predict_tail(PredictSmem& sm, const PredictArgs& a, const PrCta& q, int z, double sf2,
                                                double (&qf)[2], double (&mp)[2]) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        qf[h] += __shfl_xor_sync(0xffffffffu, qf[h], 1);
        qf[h] += __shfl_xor_sync(0xffffffffu, qf[h], 2);
        mp[h] += __shfl_xor_sync(0xffffffffu, mp[h], 1);
        mp[h] += __shfl_xor_sync(0xffffffffu, mp[h], 2);
    }
    if (q.t == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) { sm.red[q.wc][0][q.wm + q.g + 8 * h] = qf[h]; sm.red[q.wc][1][q.wm + q.g + 8 * h] = mp[h]; }
    }
    __syncthreads();
    double* part = a.part + (((size_t)z * a.nrb + q.rb) * a.nj) * 2 * PR_TR;
    if (q.tid < 2 * PR_TR) {                                    // column warps in fixed order
        const int w = q.tid / PR_TR, r = q.tid % PR_TR;
        part[(size_t)q.jb * 2 * PR_TR + q.tid] = ((sm.red[0][w][r] + sm.red[1][w][r]) + sm.red[2][w][r]) + sm.red[3][w][r];
    }
    if (!last_cta_arrives(a.cnt + (size_t)z * a.nrb + q.rb, (unsigned)a.nj)) return;
    if (q.tid < PR_TR && q.r0 + q.tid < a.T) {                  // j blocks in fixed order
        double qs = 0.0, ms = 0.0;
        for (int b = 0; b < a.nj; ++b) { qs += part[(size_t)b * 2 * PR_TR + q.tid]; ms += part[(size_t)b * 2 * PR_TR + PR_TR + q.tid]; }
        a.mean[(size_t)(q.r0 + q.tid) * a.ne + z] = ms;
        a.var[(size_t)(q.r0 + q.tid) * a.ne + z] = sf2 - qs;
    }
}

// grid (nj, nrb, ne), 256 threads
__global__ void __launch_bounds__(256, 2) gp_predict_kernel(PredictArgs a) {
    PDL_ENTRY();
    extern __shared__ __align__(16) unsigned char pr_smem_raw[];
    PredictSmem& sm = *reinterpret_cast<PredictSmem*>(pr_smem_raw);
    const PrCta q(a.np);
    const int z = blockIdx.z, e = a.e0 + z, D = a.D;
    const double sf2 = a.sf2[e];
    pr_stage(sm.s, q, a, e);
    double acc[8][4];
    pr_main_loop(sm.s, q, a, e, pr_kstar_fill(sm.s, q, a, sf2), acc);
    // epilogue: W = K* iK[:, j block] is in acc.  Row dot with K*[rows, j block] (recomputed: same function, same bits)
    // and the mean partial K*[rows, j block] beta[j block].
    double qf[2] = {0.0, 0.0}, mp[2] = {0.0, 0.0};
    if (q.active) {
        const double* be = a.beta + (size_t)e * a.n;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = q.wm + q.g + 8 * h;
            if (q.r0 + r < a.T) {
#pragma unroll
                for (int k2 = 0; k2 < 8; ++k2)
#pragma unroll
                    for (int o = 0; o < 2; ++o) {
                        const int j = q.j0 + q.wn + 8 * k2 + 2 * q.t + o;
                        if (j < a.n) {
                            const double k = pr_kstar(&sm.s.x[r * MAXD], a.C + (size_t)j * D, sm.s.il, D, sf2);
                            qf[h] = fma(acc[k2][2 * h + o], k, qf[h]);
                            mp[h] = fma(k, be[j], mp[h]);
                        }
                    }
            }
        }
    }
    pr_predict_tail(sm, a, q, z, sf2, qf, mp);
}

// ---- VJP of the diagonal posterior at the inputs (pilco_gp_predict_vjp, DESIGN.md section 12) ----------------------
//   gx = sum_e ell_e^-2 o sum_n c_en (c_n - x),   c_en = k_en (gmean_e beta_en - 2 gvar_e w_en),   w_e = iK_e k_e
// (d k_en / dx = k_en (c_n - x) / ell_e^2; d var / d k = -2 w since iK is symmetric).  The difference form c_n - x is
// summed directly: the expanded sum_n c_n c_n - (sum_n c_n) x would cancel when |x| >> |c_n - x|.
struct VjpArgs : PrArgs {       // part: [E, nrb, nj, PR_TR, D] sums of c_en (c_n - x); cnt: [nrb] over nj * E CTAs
    int E;
    const double* gmean;        // [T,E]
    const double* gvar;         // [T,E]
    double* gXs;                // [T,D]
};

struct VjpSmem {
    PrTile s;                           // after the main loop, B holds c [PR_TR][PR_LDB]
    double gm[PR_TR], gv[PR_TR];        // the rows' cotangents of output e
};
static_assert(2 * PR_KC >= PR_TR, "c of the CTA's rows x j block fits the iK double buffer");

// VJP tail, once the kernel has written c for the CTA's (rows, j block) to the free iK buffer: 8 lanes per row sum
// c (c_n - x) over the block's columns in a fixed order and the last of the row block's nj * E CTAs applies ell_e^-2
// and sums the outputs and j blocks in a fixed order (DIR: plus the direct sums dir [E,T,D] of each output before
// ell_e^-2).  The c loop stays in the kernels: shared, with c's formula passed in, fs_predict_vjp_kernel spills.
template <bool DIR>
__device__ __forceinline__ void pr_vjp_tail(VjpSmem& sm, const VjpArgs& a, const PrCta& q, int e, const double* dir) {
    const int D = a.D;
    const double* cs = &sm.s.B[0][0];                           // c [PR_TR][PR_LDB]
    __syncthreads();
    {                                                           // row r = tid / 8; lane s sums columns s, s + 8, ...
        const int r = q.tid >> 3, s = q.tid & 7;
        const int jend = min(PR_JB, a.n - q.j0);
        const double* xr = &sm.s.x[r * MAXD];
        double gs[MAXD];
#pragma unroll
        for (int d = 0; d < MAXD; ++d) gs[d] = 0.0;
        for (int jl = s; jl < jend; jl += 8) {
            const double c = cs[r * PR_LDB + jl];
            const double* cj = a.C + (size_t)(q.j0 + jl) * D;
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < D) gs[d] = fma(c, cj[d] - xr[d], gs[d]);
        }
#pragma unroll
        for (int d = 0; d < MAXD; ++d) {                        // over the 8 lanes of a row: fixed butterfly
            gs[d] += __shfl_xor_sync(0xffffffffu, gs[d], 1);
            gs[d] += __shfl_xor_sync(0xffffffffu, gs[d], 2);
            gs[d] += __shfl_xor_sync(0xffffffffu, gs[d], 4);
        }
        if (s == 0 && q.r0 + r < a.T) {
            double* pr = a.part + ((((size_t)e * a.nrb + q.rb) * a.nj + q.jb) * PR_TR + r) * D;
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < D) pr[d] = gs[d];
        }
    }
    if (!last_cta_arrives(a.cnt + q.rb, (unsigned)(a.nj * a.E))) return;
    for (int k = q.tid; k < PR_TR * D; k += 256) {              // outputs, then j blocks (then the direct sum)
        const int r = k / D, d = k % D;
        if (q.r0 + r >= a.T) continue;
        double sum = 0.0;
        for (int ee = 0; ee < a.E; ++ee) {
            const double* pe = a.part + (((size_t)ee * a.nrb + q.rb) * a.nj * PR_TR + r) * D + d;
            double se = 0.0;
            for (int b = 0; b < a.nj; ++b) se += pe[(size_t)b * PR_TR * D];
            if (DIR) se += dir[((size_t)ee * a.T + q.r0 + r) * D + d];
            const double il = 1.0 / a.ell[(size_t)ee * D + d];
            sum = fma(se, il * il, sum);
        }
        a.gXs[(size_t)(q.r0 + r) * D + d] = sum;
    }
}

// grid (nj, nrb, E), 256 threads.  The main loop is gp_predict_kernel's (W = K* iK[:, j block]).
__global__ void __launch_bounds__(256, 2) gp_predict_vjp_kernel(VjpArgs a) {
    PDL_ENTRY();
    extern __shared__ __align__(16) unsigned char pr_smem_raw[];
    VjpSmem& sm = *reinterpret_cast<VjpSmem*>(pr_smem_raw);
    const PrCta q(a.np);
    const int e = blockIdx.z;
    const double sf2 = a.sf2[e];
    if (q.tid < PR_TR) {
        const bool in = q.r0 + q.tid < a.T;
        sm.gm[q.tid] = in ? a.gmean[(size_t)(q.r0 + q.tid) * a.E + e] : 0.0;
        sm.gv[q.tid] = in ? a.gvar[(size_t)(q.r0 + q.tid) * a.E + e] : 0.0;
    }
    pr_stage(sm.s, q, a, e);
    double acc[8][4];
    pr_main_loop(sm.s, q, a, e, pr_kstar_fill(sm.s, q, a, sf2), acc);
    __syncthreads();                                            // every warp is done with the last iK tile
    double* cs = &sm.s.B[0][0];                                 // c [PR_TR][PR_LDB]
    const double* be = a.beta + (size_t)e * a.n;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = q.wm + q.g + 8 * h;
#pragma unroll
        for (int k2 = 0; k2 < 8; ++k2)
#pragma unroll
            for (int o = 0; o < 2; ++o) {
                const int jl = q.wn + 8 * k2 + 2 * q.t + o, j = q.j0 + jl;
                double c = 0.0;
                if (q.active && q.r0 + r < a.T && j < a.n) {
                    const double k = pr_kstar(&sm.s.x[r * MAXD], a.C + (size_t)j * a.D, sm.s.il, a.D, sf2);
                    c = k * fma(-2.0 * sm.gv[r], acc[k2][2 * h + o], sm.gm[r] * be[j]);
                }
                cs[r * PR_LDB + jl] = c;
            }
    }
    pr_vjp_tail<false>(sm, a, q, e, nullptr);
}

// ---- predict for the consistent particle sampler (pilco_particles_rollout_consistent, DESIGN.md section 14) ---------
// gp_predict_kernel with two extra epilogue stores of values it already holds: W = K* iK (the C fragments) to
// W[e, row, :] and the recomputed K* to Ks[e, row, :], both [ne, T, np] with zeros past n.  mean and var are bitwise
// those of pilco_gp_predict at the same inputs (same main loop, same epilogue order, same reduction tail).
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
    const PrCta q(a.np);
    const int z = blockIdx.z, e = a.e0 + z, D = a.D;
    const double sf2 = a.sf2[e];
    pr_stage(sm.s, q, a, e);
    double acc[8][4];
    pr_main_loop(sm.s, q, a, e, pr_kstar_fill(sm.s, q, a, sf2), acc);
    // epilogue.  W (0 past n) goes to the free iK buffer and out to global memory as coalesced 16-byte rows; then
    // gp_predict_kernel's sums in its order, with each thread's W entries read back from the buffer (the same values)
    // and overwritten by K*, which goes out the same way.
    __syncthreads();                                            // every warp is done with the last iK tile
    double* cs = &sm.s.B[0][0];                                 // [PR_TR][PR_LDB]
    const int jw2 = q.jw >> 1;
    auto store_tile = [&](double* dst) {                        // cs rows < T, columns [0, jw) -> dst[z, r0 + r, j0 ..]
        for (int i = q.tid; i < PR_TR * jw2; i += 256) {
            const int r = i / jw2, c2 = i % jw2;
            if (q.r0 + r < a.T)
                *reinterpret_cast<double2*>(dst + ((size_t)z * a.T + q.r0 + r) * a.np + q.j0 + 2 * c2) =
                    *reinterpret_cast<const double2*>(cs + r * PR_LDB + 2 * c2);
        }
    };
    if (q.active) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int k2 = 0; k2 < 8; ++k2)
#pragma unroll
                for (int o = 0; o < 2; ++o) {
                    const int jl = q.wn + 8 * k2 + 2 * q.t + o;
                    cs[(q.wm + q.g + 8 * h) * PR_LDB + jl] = q.j0 + jl < a.n ? acc[k2][2 * h + o] : 0.0;
                }
    }
    __syncthreads();
    store_tile(fa.W);
    __syncthreads();                                            // W is out before K* overwrites it
    double qf[2] = {0.0, 0.0}, mp[2] = {0.0, 0.0};
    if (q.active) {
        const double* be = a.beta + (size_t)e * a.n;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = q.wm + q.g + 8 * h;
            if (q.r0 + r < a.T) {
                for (int k2 = 0; k2 < 8; ++k2)
#pragma unroll
                    for (int o = 0; o < 2; ++o) {
                        const int j = q.j0 + q.wn + 8 * k2 + 2 * q.t + o;
                        double* c = &cs[r * PR_LDB + q.wn + 8 * k2 + 2 * q.t + o];
                        double k = 0.0;
                        if (j < a.n) {
                            k = pr_kstar(&sm.s.x[r * MAXD], a.C + (size_t)j * D, sm.s.il, D, sf2);
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
    pr_predict_tail(sm, a, q, z, sf2, qf, mp);
}

// ---- VJP for the gradient of the consistent sampler (pilco_particles_rollout_consistent_grad, DESIGN.md section 15) --
//   gx = sum_e ell_e^-2 o (sum_n c_en (c_n - x) + dir_e),   c_en = k_en (gmean_e beta_en + [a_e iK_e]_n)
// gp_predict_vjp_kernel with the row a_e (fs_cond_bwd_kernel: -2 var_bar K* - sum_s G_s K*_s) as the A operand of the
// main loop instead of K*, so the contraction gives a iK directly, and the per-output direct sums dir_e of the
// cross-covariance terms added by the last-arriving CTA before ell_e^-2.
struct FsVjpArgs {
    VjpArgs v;                  // gvar unused: it is folded into A
    const double* A;            // [E, T, np]  a rows, zeros past n
    const double* dir;          // [E, T, D]   direct sums
};

// grid (nj, nrb, E), 256 threads: gp_predict_vjp_kernel's decomposition
__global__ void __launch_bounds__(256, 2) fs_predict_vjp_kernel(FsVjpArgs fa) {
    PDL_ENTRY();
    const VjpArgs& a = fa.v;
    extern __shared__ __align__(16) unsigned char pr_smem_raw[];
    VjpSmem& sm = *reinterpret_cast<VjpSmem*>(pr_smem_raw);
    const PrCta q(a.np);
    const int e = blockIdx.z;
    const double sf2 = a.sf2[e];
    const double* Ae = fa.A + (size_t)e * a.T * a.np;
    if (q.tid < PR_TR) sm.gm[q.tid] = q.r0 + q.tid < a.T ? a.gmean[(size_t)(q.r0 + q.tid) * a.E + e] : 0.0;
    pr_stage(sm.s, q, a, e);
    auto achunk = [&](double* A, int c) {                       // a[rows, c KC .. (c+1) KC); 0 past n or T
        for (int k2 = q.tid; k2 < PR_TR * PR_KC; k2 += 256) {
            const int r = k2 / PR_KC, k = k2 % PR_KC, i = c * PR_KC + k;
            A[r * PR_LDA + k] = (i < a.n && q.r0 + r < a.T) ? Ae[(size_t)(q.r0 + r) * a.np + i] : 0.0;
        }
    };
    double acc[8][4];
    pr_main_loop(sm.s, q, a, e, achunk, acc);
    __syncthreads();                                            // every warp is done with the last iK tile
    double* cs = &sm.s.B[0][0];                                 // c [PR_TR][PR_LDB]
    const double* be = a.beta + (size_t)e * a.n;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int r = q.wm + q.g + 8 * h;
#pragma unroll
        for (int k2 = 0; k2 < 8; ++k2)
#pragma unroll
            for (int o = 0; o < 2; ++o) {
                const int jl = q.wn + 8 * k2 + 2 * q.t + o, j = q.j0 + jl;
                double c = 0.0;
                if (q.active && q.r0 + r < a.T && j < a.n) {
                    const double k = pr_kstar(&sm.s.x[r * MAXD], a.C + (size_t)j * a.D, sm.s.il, a.D, sf2);
                    c = k * fma(sm.gm[r], be[j], acc[k2][2 * h + o]);
                }
                cs[r * PR_LDB + jl] = c;
            }
    }
    pr_vjp_tail<true>(sm, a, q, e, fa.dir);
}

// ---- host side ------------------------------------------------------------------------------------------------------
// A call's workspace: the partial sums, then the arrival counters (16-byte aligned).  pr_diag_ws and pr_vjp_ws are the
// only places that know the layout: the byte count and the pointers come from the same function.
struct PrWs { int nj, nrb; size_t ncnt, bytes; double* part; unsigned* cnt; };

static PrWs pr_ws(int np, int T, size_t part_per_cta, size_t cnt_per_rb, void* ws) {
    PrWs w;
    w.nj = (np + PR_JB - 1) / PR_JB; w.nrb = (T + PR_TR - 1) / PR_TR;
    const size_t part = part_per_cta * w.nrb * w.nj * sizeof(double);
    w.ncnt = cnt_per_rb * w.nrb;
    w.bytes = part + ((w.ncnt * sizeof(unsigned) + 15) & ~(size_t)15);
    w.part = (double*)ws;
    w.cnt = ws ? (unsigned*)((char*)ws + part) : nullptr;
    return w;
}
// diagonal predict of ne outputs: part [ne, nrb, nj, 2, PR_TR], cnt [ne, nrb]
static PrWs pr_diag_ws(int np, int ne, int T, void* ws = nullptr) { return pr_ws(np, T, (size_t)ne * 2 * PR_TR, ne, ws); }
// VJP over E outputs: part [E, nrb, nj, PR_TR, D], cnt [nrb]
static PrWs pr_vjp_ws(int np, int D, int E, int T, void* ws = nullptr) { return pr_ws(np, T, (size_t)E * PR_TR * D, 1, ws); }

static PrArgs pr_args(const pilco_gp_model* gp, int T, const double* Xs, const PrWs& w) {
    PrArgs a;
    a.n = gp->n; a.D = gp->D; a.np = pad64(gp->n); a.nj = w.nj; a.nrb = w.nrb; a.T = T;
    a.C = gp->X; a.ell = gp->ell; a.sf2 = gp->sf2; a.beta = gp->beta; a.iK = gp->iK; a.ldk = gp->ldk;
    a.Xs = Xs; a.part = w.part; a.cnt = w.cnt;
    return a;
}

// zero the counters and launch K on grid (nj, nrb, nz), 256 threads
template <auto K, size_t SMEM, class Args>
static int pr_launch(cudaStream_t st, const PrWs& w, int nz, const Args& a) {
    if (const int rc = pilco_smem_optin<K>((int)SMEM)) return rc;
    cudaMemsetAsync(w.cnt, 0, w.ncnt * sizeof(unsigned), st);
    const dim3 grid(w.nj, w.nrb, nz);
    launch_pri(pilco_small_grid(grid), K, grid, dim3(256), SMEM, st, a);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

// the consistent rollout and its gradient set the attributes before they enqueue anything
int fs_predict_prepare() { return pilco_smem_optin<fs_predict_kernel>((int)sizeof(PredictSmem)); }
int fs_vjp_prepare() { return pilco_smem_optin<fs_predict_vjp_kernel>((int)sizeof(VjpSmem)); }

// all ne = E outputs of the validated model at T points (T <= 65535 * PR_TR); ws: pilco_gp_predict's diagonal workspace
int fs_predict_launch(cudaStream_t st, const pilco_gp_model* gp, int T, const double* Xs, double* mean, double* var,
                      double* W, double* Ks, void* ws) {
    const PrWs w = pr_diag_ws(pad64(gp->n), gp->E, T, ws);
    FsPredArgs fa;
    static_cast<PrArgs&>(fa.p) = pr_args(gp, T, Xs, w);
    fa.p.e0 = 0; fa.p.ne = gp->E; fa.p.mean = mean; fa.p.var = var;
    fa.W = W; fa.Ks = Ks;
    return pr_launch<fs_predict_kernel, sizeof(PredictSmem)>(st, w, gp->E, fa);
}

// d/dXs of the validated model at T points given gmean [T,E], the a rows [E,T,np] and the direct sums [E,T,D];
// ws: pilco_gp_predict_vjp's workspace at T
int fs_vjp_launch(cudaStream_t st, const pilco_gp_model* gp, int T, const double* Xs, const double* gmean,
                  const double* A, const double* dir, double* gXs, void* ws) {
    const PrWs w = pr_vjp_ws(pad64(gp->n), gp->D, gp->E, T, ws);
    FsVjpArgs fa;
    static_cast<PrArgs&>(fa.v) = pr_args(gp, T, Xs, w);
    fa.v.E = gp->E; fa.v.gmean = gmean; fa.v.gvar = nullptr; fa.v.gXs = gXs;
    fa.A = A; fa.dir = dir;
    return pr_launch<fs_predict_vjp_kernel, sizeof(VjpSmem)>(st, w, gp->E, fa);
}

// full covariance (factorize.cu): K*, K** (gram_kernel), W = K* iK, K** - W K*' and K* beta (gemm)
int gp_predict_full_cov(cudaStream_t st, int n, int D, int ne, int T, const double* C, const double* ell, const double* sf2,
                        const double* beta, const double* iK, int ldk, const double* Xs, double* mean, double* cov, double* ws);

extern "C" {

size_t pilco_gp_predict_workspace_bytes(int n, int D, int E, int T, int full_cov) {
    if (n < 1 || D < 1 || D > MAXD || E < 1 || E > MAXE || T < 1 || T > 65535 * PR_TR) return 0;
    const int np = pad64(n);
    if (full_cov) return T > 65535 * 8 ? 0 : 2 * (size_t)E * T * np * sizeof(double);    // K*, W = K* iK  [E,T,np] each
    return pr_diag_ws(np, E, T).bytes;
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
    const PrWs w = pr_diag_ws(pad64(n), ne, T, ws);
    PredictArgs a;
    static_cast<PrArgs&>(a) = pr_args(gp, T, Xs, w);
    a.e0 = e0; a.ne = ne; a.mean = mean; a.var = var;
    return pr_launch<gp_predict_kernel, sizeof(PredictSmem)>(st, w, ne, a);
}

size_t pilco_gp_predict_vjp_workspace_bytes(int n, int D, int E, int T) {
    if (n < 1 || D < 1 || D > MAXD || E < 1 || E > MAXE || T < 1 || T > 65535 * PR_TR) return 0;
    return pr_vjp_ws(pad64(n), D, E, T).bytes;
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
    const PrWs w = pr_vjp_ws(pad64(n), D, E, T, ws);
    VjpArgs a;
    static_cast<PrArgs&>(a) = pr_args(gp, T, Xs, w);
    a.E = E; a.gmean = gmean; a.gvar = gvar; a.gXs = gXs;
    return pr_launch<gp_predict_vjp_kernel, sizeof(VjpSmem)>((cudaStream_t)stream, w, E, a);
}

}  // extern "C"
