// mm_kernels.cuh -- device side of the fused SE-ARD moment match (forward).
//
// Algorithm (per batch element r; see DESIGN.md "Moment-match kernels"):
//   setup   grid (E + P, R): output tasks a<E   : W_a=(s+diag ell_a^2)^-1 (Cholesky), mean M_a, V_a
//                            pair tasks (a<=b)  : Q_ab = 0.5 R^-1 s via chol(s+diag(1/(p_a+p_b))),
//                                                 per-centre A'_ab[n], B_ab[n], U'_ab[n][:]
//   tile    grid (NB, P, R): T_ab = sum_{n,m} (beta_a[n] beta_b[m] - d_ab iK_a[n,m])
//                                              * exp(A'[n] + B[m] + U'[n].zeta[m])
//                            off-diagonal pairs: 16 rows per warp, one 16x8 MMA per K chunk for U'.zeta
//                            (mm_tile_m16_kernel); diagonal pairs: 8 rows per warp, DMMA m8n8k4; table exp, TMA-staged columns
//   finish  grid (R)       : S_ab = T_ab + d_ab*diag_add - M_a M_b
// Reference: pilco/models/mgpr.py:91-149 (gp0.m:63-104, gp2.m:69-106).
#pragma once
#include "common.cuh"
#include <type_traits>

#define TILE_CM 512        // columns staged in shared memory per chunk
// per-pair constants written by setup stage 1: Qa = Q diag(p_a) [MAXD*MAXD], Qb = Q diag(p_b), p_a, p_b,
// 0.5 log det R, log sf2_a, log sf2_b
#define PAIR_QA 0
#define PAIR_QB (MAXD * MAXD)
#define PAIR_PA (2 * MAXD * MAXD)
#define PAIR_PB (2 * MAXD * MAXD + MAXD)
#define PAIR_SC (2 * MAXD * MAXD + 2 * MAXD)
#define PAIR_BLK (2 * MAXD * MAXD + 2 * MAXD + 8)

struct MMWs {            // workspace layout, offsets in doubles relative to the per-restart base
    size_t zeta, betap, Bq, Tpart, Wm, Wc, Qab, Ufrag, Arow, per_r;
    int np, ldz, P, NB;
};

static inline __host__ __device__ MMWs mm_ws_layout(int n, int D, int E, bool ordered = false) {
    MMWs L;
    L.np = pad64(n); L.ldz = ldz_of(D); L.P = ordered ? E * E : npairs_of(E); L.NB = L.np / 64;
    size_t o = 0;
    L.zeta = o;  o += (size_t)L.np * L.ldz;
    L.betap = o; o += (size_t)E * L.np;
    L.Bq = o;    o += (size_t)L.P * L.np;
    L.Tpart = o; o += (size_t)L.P * (L.np / 8);
    o = (o + 1) & ~(size_t)1;
    L.Wm = o;    o += (size_t)E * MAXD * MAXD;          // setup stage 1 -> 2: W_a
    L.Wc = o;    o += (size_t)((E + 1) & ~1);           //                      c_a
    L.Qab = o;   o += (size_t)L.P * PAIR_BLK;           //                      per-pair block (see PAIR_*)
    o = (o + 1) & ~(size_t)1;
    // forward (unordered pairs): row-side operands of every (pair, row octet) materialised by setup stage 2 so that
    // the tile CTAs start their column sweep after one round of loads -- U' as DMMA A fragments
    // [P][np/8][KS][32 lanes] and the scalar A'[P][np].  The backward tile kernel derives them in its prologue.
    L.Ufrag = o; if (!ordered) o += (size_t)L.P * (L.np / 8) * ksteps_of(D) * 32;
    L.Arow = o;  if (!ordered) o += (size_t)L.P * L.np;
    L.per_r = (o + 1) & ~(size_t)1;
    return L;
}

// layout of the tape of one taped moment-match call (mm_tape.cuh), offsets in doubles per restart
struct MMTapeL { size_t Q, C, Ld, hr, hc, HZ, per_r; int cs, ldh, np, P; };

struct MMParams {
    pilco_gp_model gp;
    int R;
    const double* m; const double* s;      // [R] rows with strides m_rs / s_rs (doubles)
    long long m_rs, s_rs;
    double* M; double* S; double* V;
    int* info;
    double* ws;
    MMWs L;
    // backward-mode setup (ordered pairs q = a*E + b): also store Q_ab, C_ab=(s+diag(1/delta))^-1 and
    // logdet R_ab per pair; offsets (doubles, per restart) of those arrays inside ws.  bwd==0: unused.
    int bwd;
    size_t oQ, oC, oLd;
    // taped forward (mm_tape.cuh): tape != nullptr -> setup stage 1 also stores Q, C, logdet R per unordered pair and
    // the taped tile kernel runs in place of mm_tile_kernel
    double* tape = nullptr;
    MMTapeL TL;
};

// the parameter block of one forward moment match on the forward workspace layout; with a tape, the taped tile pass
// writing tape layout TL.  Value-initialised: the backward-mode fields and TL are defined whatever the caller sets.
static inline MMParams mm_params(const pilco_gp_model* gp, int R, const double* m, long long m_rs, const double* s,
                                 long long s_rs, double* M, double* S, double* V, int* info, double* ws,
                                 double* tape = nullptr, const MMTapeL& TL = MMTapeL()) {
    MMParams p{};
    p.gp = *gp; p.R = R; p.m = m; p.m_rs = m_rs; p.s = s; p.s_rs = s_rs; p.M = M; p.S = S; p.V = V; p.info = info;
    p.ws = ws; p.L = mm_ws_layout(gp->n, gp->D, gp->E); p.tape = tape; p.TL = TL;
    return p;
}

// The launch decisions that follow the batch size and the machine, as functions of (shape, R, SMs) so that the host
// suite can say which kernel branch a given case runs (tests/mm_cases.py).
//
// Row blocks per forward tile CTA: a CTA's fixed cost (TMA staging of the columns and the exp table, barrier,
// first-load latency: ~5 k cycles against ~16 k per 64-row sweep at the metric shape) is paid once for all its row
// blocks.  All NB row blocks of a pair go to one CTA as soon as pairs x restarts still give every SM a CTA; smaller
// launches keep enough CTAs to fill the machine (2 CTAs per SM).
static inline int mm_tile_rpc(int NB, int P, int R, int nsm) {
    const long long pr = (long long)P * R;
    if (pr >= nsm) return NB;
    const int rpc = (int)(((long long)NB * pr) / (2LL * nsm));
    return rpc < 1 ? 1 : rpc;
}
// Both setup stages in ONE launch while the whole launch is small -- at most half the SMs' worth of CTAs: a single
// restart, or the RBF policy's few tasks (see mm_setup_launch)
static inline bool mm_setup_is_fused(int ntask, int R, int nsm) { return (long long)ntask * R <= nsm / 2; }
// Row splits of one pair over the CTAs of the taped tile kernel (mm_tape.cuh): 1 once pairs x restarts fill the machine
// twice over, at most 4, and never fewer than 8 row octets per split
static inline int mm_tape_splits_on(int n, int P, int R, int nsm) {
    const int NO = (n + 7) / 8;
    const long long pr = (long long)P * R, fill = 2LL * nsm;
    int cs = 1;
    if (pr < fill) cs = (int)((fill + pr - 1) / pr);
    int cap = NO / 8;
    if (cap < 1) cap = 1;
    if (cap > 4) cap = 4;
    return cs < cap ? cs : cap;
}


#ifdef __CUDACC__

// -------------------------------------------------------------------------------------------------
// setup: ONE WARP PER TASK (4 tasks per CTA).  The D x D Cholesky runs in registers (lane i owns row i,
// column broadcasts by shuffle), the triangular solves keep each right-hand side in registers and read
// L from per-warp shared memory, the per-centre loop strides the 32 lanes over the centres.
// -------------------------------------------------------------------------------------------------
#define SETUP_WARPS 4

// lane i (< DP) holds row i of the SPD matrix in a[0..DP); on exit row i of its lower Cholesky factor, with the
// INVERSE pivots 1/L[j][j] in ipd[j] (same value in every lane).  Returns false if a pivot is not positive.
template <int DP>
__device__ __forceinline__ bool chol_regs(double (&a)[DP], double (&ipd)[DP], int lane) {
    bool ok = true;
#pragma unroll
    for (int j = 0; j < DP; ++j) {
        double d = __shfl_sync(0xffffffffu, a[j], j);
        if (!(d > 0.0)) { ok = false; d = 1.0; }
        const double ip = rsqrt(d);
        ipd[j] = ip;
        const double lij = (lane == j) ? d * ip : a[j] * ip;
        a[j] = lij;
#pragma unroll
        for (int k = j + 1; k < DP; ++k) {
            const double lkj = __shfl_sync(0xffffffffu, lij, k);
            if (lane >= k) a[k] = fma(-lij, lkj, a[k]);
        }
    }
    return ok;
}

// Solve (L L^T) x = y for the right-hand side held in y[0..DP) (one per lane); L in shared memory [DP][SLD],
// inverse pivots in ipd.
template <int DP>
__device__ __forceinline__ void chol_solve_regs(const double* __restrict__ Ls, const double (&ipd)[DP], double (&y)[DP]) {
#pragma unroll
    for (int i = 0; i < DP; ++i) {
        double v = y[i];
#pragma unroll
        for (int k = 0; k < i; ++k) v = fma(-Ls[i * SLD + k], y[k], v);
        y[i] = v * ipd[i];
    }
#pragma unroll
    for (int i = DP - 1; i >= 0; --i) {
        double v = y[i];
#pragma unroll
        for (int k = i + 1; k < DP; ++k) v = fma(-Ls[k * SLD + i], y[k], v);
        y[i] = v * ipd[i];
    }
}

// stage 1: the serial part of every task (one warp per task): D x D Cholesky + solves -> matrices in workspace
// symmetrised input covariance of restart r -> s_s [DP][SLD] (all threads of the CTA; caller synchronises)
template <int DP>
__device__ __forceinline__ void setup_stage_s(const MMParams& p, int r, double* s_s) {
    const int D = p.gp.D;
    const double* sr = p.s + (size_t)r * p.s_rs;
    for (int e = threadIdx.x; e < DP * DP; e += blockDim.x) {
        const int i = e / DP, j = e % DP;
        s_s[i * SLD + j] = (i < D && j < D) ? 0.5 * (sr[i * D + j] + sr[j * D + i]) : 0.0;
    }
}

// Is the symmetrised input covariance s_s positive semi-definite?  (one warp.)  The Cholesky of s + tau I, tau =
// PILCO_MM_PSD_TOL x the largest |s_ii|, succeeds for every PSD s (zero, singular, badly conditioned: its rounding is far
// below tau) and fails as soon as s has an eigenvalue below -tau -- an input the moment match would still evaluate to
// finite numbers, since s + diag(ell^2) stays positive definite.
template <int DP>
__device__ __forceinline__ bool setup_s_is_psd(const double* s_s, int D, int lane) {
    const int li = lane < DP ? lane : DP - 1;
    double smax = 0.0;
    for (int d = 0; d < D; ++d) smax = fmax(smax, fabs(s_s[d * SLD + d]));
    const double tau = fma(PILCO_MM_PSD_TOL, smax, 1e-300);
    double arow[DP], ipd[DP];
#pragma unroll
    for (int j = 0; j < DP; ++j) arow[j] = s_s[li * SLD + j] + (j == li ? tau : 0.0);
    return chol_regs<DP>(arow, ipd, lane);
}

// stage 1 of ONE task by ONE warp (scratch Ls, Qs [MAXD*SLD], pa, pb, dinv [MAXD] private to the warp)
template <int DP, bool BWD>
__device__ __forceinline__ void mm_setup1_task(const MMParams& p, int r, int task, int lane, const double* s_s,
                                               double* Ls, double* Qs, double* pa, double* pb, double* dinv,
                                               bool check_s = true) {
    const pilco_gp_model& gp = p.gp;
    const int D = gp.D, E = gp.E;
    const MMWs& L = p.L;
    const double* ell = gp.ell + (size_t)r * gp.ell_bs;
    const double* sf2 = gp.sf2 + (size_t)r * gp.sf2_bs;
    double* wsr = p.ws + (size_t)r * L.per_r;
    const int li = lane < DP ? lane : DP - 1;                  // clamp so idle lanes read valid memory

    if (!BWD && task < E) {
        // ---------------- output task: W_a = (s + Lambda_a^2)^-1 and c_a ----------------
        const int a = task;
        const double l = lane < D ? ell[a * D + lane] : 1.0;
        const bool lbad = !(l > 0.0 && l < INFINITY);          // a length-scale outside (0, inf): reported, never used silently
        if (lane < DP) pa[lane] = l * l;
        __syncwarp();
        double arow[DP], ipd[DP];
        // once per restart: is s itself positive semi-definite?  (two-stage form: a warp of its own, see mm_setup1_kernel)
        const bool sbad = check_s && a == 0 && !setup_s_is_psd<DP>(s_s, D, lane);
#pragma unroll
        for (int j = 0; j < DP; ++j) arow[j] = s_s[li * SLD + j] + (j == li ? pa[li] : 0.0);
        const bool ok = chol_regs<DP>(arow, ipd, lane) && !sbad && !__any_sync(0xffffffffu, lbad);
        if (lane < DP) {
#pragma unroll
            for (int j = 0; j < DP; ++j) Ls[lane * SLD + j] = arow[j];
        }
        __syncwarp();
        double y[DP];
#pragma unroll
        for (int i = 0; i < DP; ++i) y[i] = (i == li) ? 1.0 : 0.0;
        chol_solve_regs<DP>(Ls, ipd, y);                       // column `lane` of W (symmetric)
        double* Wo = wsr + L.Wm + (size_t)a * MAXD * MAXD;
        if (lane < DP) {
#pragma unroll
            for (int i = 0; i < DP; ++i) Wo[i * DP + lane] = y[i];
        }
        double pip = 1.0, pl = 1.0;                            // prod 1/L_jj, prod ell_d^2 (D <= 16: no overflow)
#pragma unroll
        for (int j = 0; j < DP; ++j) pip *= ipd[j];
        for (int d = 0; d < D; ++d) pl *= pa[d];
        if (lane == 0) {
            wsr[L.Wc + a] = sf2[a] * sqrt(pl) * pip;           // c_a = sf2 sqrt(prod ell^2 / det(s + Lambda^2))
            if (!ok && p.info) atomicOr(&p.info[r], 1);
        }
        const double* beta = gp.beta + (size_t)r * gp.beta_bs; // betap row a: beta_a zero-padded to np (tile kernels' columns)
        for (int nn = lane; nn < L.np; nn += 32) wsr[L.betap + (size_t)a * L.np + nn] = nn < gp.n ? beta[(size_t)a * gp.n + nn] : 0.0;
        return;
    }

    // ---------------- pair task: Q_ab ----------------
    const int q = task - E;
    int a, b;
    if (BWD) { a = q / E; b = q % E; } else pair_decode(q, a, b);
    const double la = lane < D ? ell[a * D + lane] : 1.0, lb = lane < D ? ell[b * D + lane] : 1.0;
    const bool lbad = !(la > 0.0 && la < INFINITY && lb > 0.0 && lb < INFINITY);
    if (lane < DP) {
        pa[lane] = lane < D ? 1.0 / (la * la) : 0.0;
        pb[lane] = lane < D ? 1.0 / (lb * lb) : 0.0;
        dinv[lane] = lane < D ? 1.0 / (1.0 / (la * la) + 1.0 / (lb * lb)) : 0.0;      // 1/(p_a+p_b)
    }
    __syncwarp();
    double arow[DP];
#pragma unroll
    for (int j = 0; j < DP; ++j) arow[j] = s_s[li * SLD + j] + (j == li ? (li < D ? dinv[li] : 1.0) : 0.0);
    double ipd[DP];
    const bool ok = chol_regs<DP>(arow, ipd, lane) && !__any_sync(0xffffffffu, lbad);
    if (lane < DP) {
#pragma unroll
        for (int j = 0; j < DP; ++j) Ls[lane * SLD + j] = arow[j];
    }
    __syncwarp();
    double y[DP];
#pragma unroll
    for (int i = 0; i < DP; ++i) y[i] = s_s[i * SLD + li];     // column `lane` of s
    chol_solve_regs<DP>(Ls, ipd, y);                           // column `lane` of (s + Dd^-1)^-1 s
    if (lane < DP) {                                           // Qraw[i][lane] = 0.5 dinv[i] y[i]
#pragma unroll
        for (int i = 0; i < DP; ++i) Qs[i * SLD + lane] = 0.5 * dinv[i] * y[i];
    }
    double pip = 1.0, pdl = 1.0;
#pragma unroll
    for (int j = 0; j < DP; ++j) pip *= ipd[j];
    for (int d = 0; d < D; ++d) pdl *= (pa[d] + pb[d]);
    const double ldet = log(pdl) - 2.0 * log(pip);             // log det R_ab = log det(s+Dd^-1) + sum log delta
    __syncwarp();
    double qsym[DP];
#pragma unroll
    for (int i = 0; i < DP; ++i) qsym[i] = 0.5 * (Qs[i * SLD + li] + Qs[li * SLD + i]);
    // stage-2 operands: Qa = Q diag(p_a), Qb = Q diag(p_b) (column `lane`), and 0.5 log det R
    double* Qo2 = wsr + L.Qab + (size_t)q * PAIR_BLK;
    if (lane < DP) {
#pragma unroll
        for (int i = 0; i < DP; ++i) { Qo2[PAIR_QA + i * DP + lane] = qsym[i] * pa[lane]; Qo2[PAIR_QB + i * DP + lane] = qsym[i] * pb[lane]; }
    }
    if (lane < MAXD) { Qo2[PAIR_PA + lane] = lane < DP ? pa[lane] : 0.0; Qo2[PAIR_PB + lane] = lane < DP ? pb[lane] : 0.0; }
    if (lane == 0) {
        Qo2[PAIR_SC + 0] = 0.5 * ldet;
        Qo2[PAIR_SC + 1] = log(sf2[a]);
        Qo2[PAIR_SC + 2] = log(sf2[b]);
        if (!ok && p.info) atomicOr(&p.info[r], 1);
    }
    if (BWD || p.tape != nullptr) {
        double* tpr = BWD ? nullptr : p.tape + (size_t)r * p.TL.per_r;
        double* Qo = BWD ? wsr + p.oQ + (size_t)q * D * D : tpr + p.TL.Q + (size_t)q * D * D;
        double* Co = BWD ? wsr + p.oC + (size_t)q * D * D : tpr + p.TL.C + (size_t)q * D * D;
        double c[DP];
#pragma unroll
        for (int i = 0; i < DP; ++i) c[i] = (i == li) ? 1.0 : 0.0;
        chol_solve_regs<DP>(Ls, ipd, c);                       // column `lane` of C = (s + Dd^-1)^-1 (symmetric)
        if (lane < D) {
#pragma unroll
            for (int i = 0; i < DP; ++i)
                if (i < D) { Qo[i * D + lane] = qsym[i]; Co[i * D + lane] = c[i]; }
        }
        if (lane == 0) { if (BWD) wsr[p.oLd + q] = ldet; else tpr[p.TL.Ld + q] = ldet; }
    }
}

// zeta = X - m of restart r ([np][ldz], zero outside rows [0, n) and columns [0, D)) with coalesced 16-byte stores:
// thread `first` of the `stride` threads writing it takes every stride-th 16-byte pair (forward mode: once per restart)
template <int DP>
__device__ __forceinline__ void setup_publish_zeta(const MMParams& p, int r, int first, int stride) {
    constexpr int ldz = DP <= 4 ? 4 : (DP <= 12 ? 12 : 20);   // == L.ldz
    const int n = p.gp.n, D = p.gp.D;
    const double* X = p.gp.X + (size_t)r * p.gp.X_bs;
    const double* mr = p.m + (size_t)r * p.m_rs;
    double2* dst = reinterpret_cast<double2*>(p.ws + (size_t)r * p.L.per_r + p.L.zeta);
    for (int e = first; e < p.L.np * ldz / 2; e += stride) {
        const int rr = (2 * e) / ldz, cc = (2 * e) % ldz;
        const double z0 = (rr < n && cc < D) ? X[(size_t)rr * D + cc] - mr[cc] : 0.0;
        const double z1 = (rr < n && cc + 1 < D) ? X[(size_t)rr * D + cc + 1] - mr[cc + 1] : 0.0;
        dst[e] = make_double2(z0, z1);
    }
}

// stage 1 as its own launch (the two-stage form of mm_setup_launch).  Forward mode: output tasks also write their betap
// row, and all CTAs of the restart share writing zeta -- both read by stage 2 and the tile kernels.
template <int DP, bool BWD>
__global__ void __launch_bounds__(32 * SETUP_WARPS) mm_setup1_kernel(MMParams p) {
    PDL_ENTRY();
    const int r = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // forward mode: the last CTA holds no task -- its warp 0 checks that s is positive semi-definite, beside the tasks
    // instead of in front of one of them
    const bool checker = !BWD && blockIdx.x == gridDim.x - 1;
    const int ntask = checker ? 0 : (BWD ? p.L.P : p.gp.E + p.L.P);
    const int task0 = blockIdx.x * SETUP_WARPS + warp;
    const int task = BWD ? task0 + p.gp.E : task0;             // BWD: pair tasks only (ordered pairs)
    __shared__ double s_s[MAXD * SLD];                         // symmetrised input covariance (all warps)
    __shared__ double sLw[SETUP_WARPS][MAXD * SLD];            // per warp: Cholesky factor
    __shared__ double sQw[SETUP_WARPS][MAXD * SLD];            // per warp: raw Q
    __shared__ double spw[SETUP_WARPS][3][MAXD];
    setup_stage_s<DP>(p, r, s_s);
    __syncthreads();
    if (task0 < ntask)
        mm_setup1_task<DP, BWD>(p, r, task, lane, s_s, sLw[warp], sQw[warp], spw[warp][0], spw[warp][1], spw[warp][2], false);
    if (checker && warp == 0 && !setup_s_is_psd<DP>(s_s, p.gp.D, lane) && lane == 0 && p.info) atomicOr(&p.info[r], 1);
    if (!BWD) setup_publish_zeta<DP>(p, r, blockIdx.x * blockDim.x + tid, gridDim.x * blockDim.x);
}

// Row-side operands of a warp's row octets for the pair block `blk`: DMMA A fragments ua[ks] = U'[row][4ks+t] with
// U' = 2 EXP_SC p_b o (Qa zeta_row), and the scalar A'[row] = EXP_SC (log sf2_a - 0.5 sum p_a zeta^2 + z_a'Q z_a
// - 0.5 log det R).  2*ceil(DP/8)*KS DMMA + ONE quad reduction per 8 rows (no layout shuffles: permuted B fragments).  The pair constants (this lane's B fragments
// of Qa and its slices of p_a, p_b) are loaded once (RowOpConsts) and reused for every row octet.
template <int KS>
struct RowOpConsts {
    static constexpr int DP = 4 * KS, NT = (DP + 7) / 8;
    // B fragments of Qa with PERMUTED columns: column c of n-tile nt is Qa row 8 nt + pi(c), pi = (0,4,1,5,2,6,3,7), so
    // that the C fragment of Z.Qa' (row g; this lane's two columns = actual columns 8 nt + t and 8 nt + 4 + t) IS the
    // A-fragment layout of k-steps 2 nt and 2 nt + 1 -- U' leaves the product without a single shuffle (the same
    // trick as the taped tile kernel's second product)
    double bq[KS][NT];
    double pak[KS];             // p_a[4 ks + t]
    double pac[NT][2], pbc[NT][2];   // p_a, p_b at this lane's C-fragment columns 8 nt + t, 8 nt + 4 + t
    double lsa, hld;            // log sf2_a, 0.5 log det R
    __device__ __forceinline__ void load(const double* __restrict__ blk, int lane) {
        const int g = lane >> 2, t = lane & 3;
        const int pg = (g >> 1) | ((g & 1) << 2);              // pi(g)
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            pak[ks] = blk[PAIR_PA + 4 * ks + t];
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const int i = 8 * nt + pg;
                bq[ks][nt] = i < DP ? blk[PAIR_QA + i * DP + 4 * ks + t] : 0.0;
            }
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = 8 * nt + 4 * h + t;
                pac[nt][h] = c < DP ? blk[PAIR_PA + c] : 0.0;
                pbc[nt][h] = c < DP ? blk[PAIR_PB + c] : 0.0;
            }
        }
        lsa = blk[PAIR_SC + 1]; hld = blk[PAIR_SC + 0];
    }
};

// NO row octets at once (independent DMMA chains in flight; every octet's arithmetic is the same whatever NO is).
// zr[o] = zeta row of this lane's centre (row g of octet o), readable at [0, ldz)
template <int KS, int NO>
__device__ __forceinline__ void row_operands_octets(const RowOpConsts<KS>& c, const double* const (&zr)[NO], const bool (&live)[NO],
                                                    int lane, double (&ua)[NO][KS], double (&Apv)[NO]) {
    constexpr int DP = 4 * KS, NT = (DP + 7) / 8;
    const int t = lane & 3;
    double z[NO][KS], va[NO][NT][2];
    double x[NO];                                               // this lane's share of z_a'Q z_a - 0.5 sum p_a zeta^2
#pragma unroll
    for (int o = 0; o < NO; ++o) {
        x[o] = 0.0;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            z[o][ks] = zr[o][4 * ks + t];
            x[o] = fma(-0.5 * c.pak[ks] * z[o][ks], z[o][ks], x[o]);
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) { va[o][nt][0] = va[o][nt][1] = 0.0; }
    }
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int o = 0; o < NO; ++o) dmma884(va[o][nt][0], va[o][nt][1], z[o][ks], c.bq[ks][nt]);
    // va[nt][h] = (Qa zeta)[8 nt + 4 h + t] of row g: column 4 ks + t with ks = 2 nt + h, i.e. A-fragment layout already
#pragma unroll
    for (int o = 0; o < NO; ++o)
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            const int nt = ks >> 1, h = ks & 1;
            x[o] = fma(c.pac[nt][h] * z[o][ks], va[o][nt][h], x[o]);      // (zeta at that column is this lane's z[ks])
            ua[o][ks] = (2.0 * EXP_SC) * c.pbc[nt][h] * va[o][nt][h];
        }
#pragma unroll
    for (int o = 0; o < NO; ++o) x[o] += __shfl_xor_sync(0xffffffffu, x[o], 1);     // one quad reduction for both terms
#pragma unroll
    for (int o = 0; o < NO; ++o) x[o] += __shfl_xor_sync(0xffffffffu, x[o], 2);
#pragma unroll
    for (int o = 0; o < NO; ++o) Apv[o] = live[o] ? EXP_SC * (c.lsa + x[o] - c.hld) : NEG_PAD;
}

// one-shot form (backward tile kernel prologue): zeta rows are read from the workspace (L2 resident)
template <int KS>
__device__ __forceinline__ void tile_row_operands(const double* __restrict__ blk, const double* __restrict__ zeta,
                                                  int ldz, int row, bool live, int lane,
                                                  double (&ua)[KS], double& Apv) {
    RowOpConsts<KS> c;
    c.load(blk, lane);
    const double* const zr[1] = {zeta + (size_t)row * ldz};
    const bool l1[1] = {live};
    double u1[1][KS], a1[1];
    row_operands_octets<KS, 1>(c, zr, l1, lane, u1, a1);
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) ua[ks] = u1[0][ks];
    Apv = a1[0];
}

// Column-side exponent piece of NO row octets of a pair: B_ab[m] = EXP_SC (log sf2_b + z'(Q diag p_b) z - 0.5 sum p_b z^2)
// of this lane's centre (row g of octet o, zeta row zr[o]), (Q diag p_b) zeta as the DMMA mini-GEMM Z[8 x DP] . Qb^T
// with the B fragments bqb[ks][nt] = Qb[8 nt + g][4 ks + t], and one quad reduction; NEG_PAD for padding rows.  As in
// row_operands_octets, every octet's arithmetic is the same whatever NO is.
template <int KS, int NO>
__device__ __forceinline__ void pair_b_octets(const double (&bqb)[KS][(4 * KS + 7) / 8], const double* __restrict__ pb, double lsb,
                                              const double* const (&zr)[NO], const bool (&live)[NO], int lane, double (&bv)[NO]) {
    constexpr int DP = 4 * KS, NT = (DP + 7) / 8;
    const int t = lane & 3;
    double z[NO][KS], vb[NO][NT][2], kbp[NO], xb[NO];
#pragma unroll
    for (int o = 0; o < NO; ++o) {
        kbp[o] = 0.0;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            z[o][ks] = zr[o][4 * ks + t];
            kbp[o] = fma(pb[4 * ks + t] * z[o][ks], z[o][ks], kbp[o]);
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) { vb[o][nt][0] = vb[o][nt][1] = 0.0; }
    }
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int o = 0; o < NO; ++o) dmma884(vb[o][nt][0], vb[o][nt][1], z[o][ks], bqb[ks][nt]);
#pragma unroll
    for (int o = 0; o < NO; ++o) {
        double qbp = 0.0;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const int i0 = 8 * nt + 2 * t;                      // this lane's two columns of the C fragment
            if (i0 < DP) qbp = fma(pb[i0] * zr[o][i0], vb[o][nt][0], fma(pb[i0 + 1] * zr[o][i0 + 1], vb[o][nt][1], qbp));
        }
        xb[o] = fma(-0.5, kbp[o], qbp);                         // one quad reduction for both terms
    }
#pragma unroll
    for (int o = 0; o < NO; ++o) xb[o] += __shfl_xor_sync(0xffffffffu, xb[o], 1);
#pragma unroll
    for (int o = 0; o < NO; ++o) xb[o] += __shfl_xor_sync(0xffffffffu, xb[o], 2);
#pragma unroll
    for (int o = 0; o < NO; ++o) bv[o] = live[o] ? EXP_SC * (lsb + xb[o]) : NEG_PAD;
}

// Output task a, one centre: t = W_a z, w = beta_a[m] exp(-z'W_a z / 2); acc[i] += w t_i, acc[DP] += w
template <int DP>
__device__ __forceinline__ void out_centre(const double* __restrict__ sW, const double (&z)[DP], double bw, double (&acc)[DP + 1]) {
    double t[DP], e = 0.0;
#pragma unroll
    for (int i = 0; i < DP; ++i) {
        double v = 0.0;
#pragma unroll
        for (int j = 0; j < DP; ++j) v = fma(sW[i * DP + j], z[j], v);
        t[i] = v; e = fma(z[i], v, e);
    }
    const double w = bw * exp(-0.5 * e);
    acc[DP] += w;
#pragma unroll
    for (int i = 0; i < DP; ++i) acc[i] = fma(w, t[i], acc[i]);
}

// Output task a: the CTA's fixed-order reduction of the per-thread sums (thread tid of 128 holds centres tid + 128 k),
// then M_a = c_a sum w and V_a = c_a sum w W_a z
template <int DP>
__device__ __forceinline__ void out_task_store(const MMParams& p, int r, int a, double (&acc)[DP + 1], double* sred, double* sout) {
    const int tid = threadIdx.x, D = p.gp.D, E = p.gp.E;
    const double c = p.ws[(size_t)r * p.L.per_r + p.L.Wc + a];
    block_sum<DP + 1>(acc, DP + 1, sred, sout);
    if (tid == 0) p.M[(size_t)r * E + a] = c * sout[DP];
    if (tid < D) p.V[((size_t)r * D + tid) * E + a] = c * sout[tid];
}

// stage 2 of one task by one CTA of 128 threads, as the fused setup kernel runs it (both modes) and the ordered-pair
// backward mode's stage-2 launch.  The forward two-stage form splits it into mm_setup2_out_kernel and
// mm_setup2_pair_kernel (below), which run the same per-centre and per-octet arithmetic.
template <int DP, bool BWD>
__device__ __forceinline__ void mm_setup2_task(const MMParams& p, int r, int task, int part = 0, int nparts = 1) {
    const pilco_gp_model& gp = p.gp;
    const int n = gp.n, D = gp.D, E = gp.E;
    const MMWs& L = p.L;
    const int np = L.np;
    constexpr int ldz = DP <= 4 ? 4 : (DP <= 12 ? 12 : 20);   // == L.ldz (ldz_of), compile-time so /,% by it are cheap
    const int tid = threadIdx.x;

    __shared__ double sQa[MAXD * MAXD], sQb[MAXD * MAXD];
    __shared__ double sm[MAXD], pb[MAXD];
    __shared__ __align__(16) double sStage[128 * (MAXD + 5)];   // [128][ldz|1] staging: X block in
    __shared__ double sred[(MAXD + 1) * 4], sout[MAXD + 1];

    const double* X = gp.X + (size_t)r * gp.X_bs;
    const double* beta = gp.beta + (size_t)r * gp.beta_bs;
    const double* mr = p.m + (size_t)r * p.m_rs;
    double* wsr = p.ws + (size_t)r * L.per_r;
    if (tid < DP) sm[tid] = tid < D ? mr[tid] : 0.0;

    if (!BWD && task < E) {
        // ---------------- output task: mean M_a and V_a (betap and zeta: stage 1) ----------------
        const int a = task;
        const double* Wg = wsr + L.Wm + (size_t)a * MAXD * MAXD;
        for (int e = tid; e < DP * DP; e += blockDim.x) sQa[e] = Wg[e];
        __syncthreads();
        double acc[DP + 1];
#pragma unroll
        for (int i = 0; i <= DP; ++i) acc[i] = 0.0;
        const int lds = ldz | 1;
        for (int n0 = 0; n0 < n; n0 += 128) {
            const int rows = (n - n0) < 128 ? (n - n0) : 128;
            __syncthreads();
            for (int e = tid; e < rows * ldz; e += blockDim.x) {
                const int rr = e / ldz, cc = e % ldz;
                if (cc < D) sStage[rr * lds + cc] = X[(size_t)(n0 + rr) * D + cc];
            }
            __syncthreads();
            const int nn = n0 + tid;
            if (nn < n) {
                double z[DP];
#pragma unroll
                for (int d = 0; d < DP; ++d) z[d] = d < D ? sStage[tid * lds + d] - sm[d] : 0.0;
                out_centre<DP>(sQa, z, beta[(size_t)a * n + nn], acc);
            }
        }
        out_task_store<DP>(p, r, a, acc, sred, sout);
        return;
    }

    // ---------------- pair task: column-side exponent piece B_ab[m] = k_b[m] + z_b' Q z_b (pre-scaled) --------
    // (Q diag p_b) zeta_m for 8 centres at a time as a small fp64-DMMA GEMM Z[8 x DP] . Qb^T.  Forward mode also
    // materialises the row-side pieces A'_ab[n], U'_ab[n] of the same 8 centres (Ufrag / Arow, read once by the
    // tile kernel); the ordered-pair backward mode leaves them to the backward tile kernel's prologue.
    const int q = task - E;
    int a, b;
    if (BWD) { a = q / E; b = q % E; } else pair_decode(q, a, b);
    constexpr int KS = DP / 4, NT = (DP + 7) / 8;
    const int lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const double* blk = wsr + L.Qab + (size_t)q * PAIR_BLK;
    for (int e = tid; e < DP * DP; e += blockDim.x) sQb[e] = blk[PAIR_QB + e];
    if (tid < MAXD) pb[tid] = blk[PAIR_PB + tid];
    __syncthreads();
    double bqb[KS][NT];                                         // B fragments: B[k][n] = Qb[n][k]
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const int i = 8 * nt + g;
            bqb[ks][nt] = i < DP ? sQb[i * DP + 4 * ks + t] : 0.0;
        }
    const double lsb = blk[PAIR_SC + 2];
    RowOpConsts<KS> roc;                                        // row-side pair constants, loaded once per CTA
    if (!BWD) roc.load(blk, lane);
    // (pair tasks may be split over `nparts` CTAs in the latency regime: CTA `part` takes every nparts-th 128-row chunk)
    for (int n0 = 128 * part; n0 < np; n0 += 128 * nparts) {
        // stage zeta[n0 : n0+128, 0:ldz] = X - m (zero outside [n, D)) in shared memory, coalesced
        __syncthreads();
        for (int e = tid; e < 128 * ldz; e += blockDim.x) {
            const int rr = e / ldz, cc = e % ldz;
            sStage[e] = (n0 + rr < n && cc < D) ? X[(size_t)(n0 + rr) * D + cc] - sm[cc] : 0.0;
        }
        __syncthreads();
        if (BWD && q == 0) {                                    // backward mode: this task also publishes zeta
            double2* dz = reinterpret_cast<double2*>(wsr + L.zeta + (size_t)n0 * ldz);
            const int rows_out = (np - n0) < 128 ? (np - n0) : 128;
            for (int e = tid; e < rows_out * ldz / 2; e += blockDim.x) dz[e] = make_double2(sStage[2 * e], sStage[2 * e + 1]);
        }
        if (BWD && b == 0) {
            const int nn = n0 + tid;
            if (nn < np) wsr[L.betap + (size_t)a * np + nn] = nn < n ? beta[(size_t)a * n + nn] : 0.0;
        }
        for (int grp = warp; grp < 16; grp += 4) {
            const int row = n0 + 8 * grp + g;
            if (n0 + 8 * grp >= np) break;                      // warp-uniform
            const double* const zr[1] = {sStage + (size_t)(8 * grp + g) * ldz};
            const bool live[1] = {row < n};
            double bv[1];
            pair_b_octets<KS, 1>(bqb, pb, lsb, zr, live, lane, bv);
            if (t == 0) wsr[L.Bq + (size_t)q * np + row] = bv[0];
            if (!BWD) {
                // row side of the same 8 centres: DMMA A fragments of U' and the scalar A' (see row_operands_octets),
                // written in the layout the tile kernel's prologue loads with three coalesced 8-byte loads per lane
                double ua[1][KS], Apv[1];
                row_operands_octets<KS, 1>(roc, zr, live, lane, ua, Apv);
                double* uf = wsr + L.Ufrag + ((size_t)q * (np >> 3) + ((n0 >> 3) + grp)) * (KS * 32);
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) uf[ks * 32 + lane] = ua[0][ks];
                if (t == 0) wsr[L.Arow + (size_t)q * np + row] = Apv[0];
            }
        }
    }
}

// stage 2 of the ordered-pair backward mode: one CTA per (ordered pair, restart)
template <int DP>
__global__ void __launch_bounds__(128) mm_setup2_bwd_kernel(MMParams p) {
    PDL_ENTRY();
    mm_setup2_task<DP, true>(p, blockIdx.y, blockIdx.x + p.gp.E);
}

// Forward stage 2, output tasks: M_a and V_a, one CTA of 128 threads per (output, restart).  The zeta rows written by
// stage 1 are read straight from the workspace (each thread's row is DP/2 contiguous 16-byte loads), one centre ahead.
// Register cap (launched with 128 threads): the prefetched row without spills, and 3 CTAs per SM at D <= 12.
template <int DP>
__global__ void __maxnreg__(DP <= 12 ? 168 : 232) mm_setup2_out_kernel(MMParams p) {
    PDL_ENTRY();
    constexpr int ldz = DP <= 4 ? 4 : (DP <= 12 ? 12 : 20);   // == L.ldz
    const int a = blockIdx.x, r = blockIdx.y, tid = threadIdx.x;
    const int n = p.gp.n;
    __shared__ double sW[DP * DP];
    __shared__ double sred[(DP + 1) * 4], sout[DP + 1];
    const double* wsr = p.ws + (size_t)r * p.L.per_r;
    const double* beta = p.gp.beta + (size_t)r * p.gp.beta_bs + (size_t)a * n;
    for (int e = tid; e < DP * DP; e += blockDim.x) sW[e] = wsr[p.L.Wm + (size_t)a * MAXD * MAXD + e];
    __syncthreads();
    double acc[DP + 1];
#pragma unroll
    for (int i = 0; i <= DP; ++i) acc[i] = 0.0;
    // thread tid takes centres tid, tid + 128, ...; the next centre's zeta row and beta are loaded before this one's sums
    const double2* zg = reinterpret_cast<const double2*>(wsr + p.L.zeta);
    double2 zn[DP / 2];
    double bn = 0.0;
    if (tid < n) {
#pragma unroll
        for (int d = 0; d < DP / 2; ++d) zn[d] = zg[(size_t)tid * (ldz / 2) + d];
        bn = beta[tid];
    }
    for (int n0 = 0; n0 < n; n0 += 128) {
        const int nn = n0 + tid;
        double z[DP];
#pragma unroll
        for (int d = 0; d < DP / 2; ++d) { z[2 * d] = zn[d].x; z[2 * d + 1] = zn[d].y; }
        const double bw = bn;
        if (nn + 128 < n) {
#pragma unroll
            for (int d = 0; d < DP / 2; ++d) zn[d] = zg[(size_t)(nn + 128) * (ldz / 2) + d];
            bn = beta[nn + 128];
        }
        __syncwarp();                                          // W stays in shared memory: it is not hoisted into DP^2 registers
        if (nn < n) out_centre<DP>(sW, z, bw, acc);
    }
    out_task_store<DP>(p, r, a, acc, sred, sout);
}

// rows of zeta per pair-kernel CTA: all np rows while zeta, the pair block and the barrier fit 48 KB of shared memory
// (np <= 448 at ldz = 12), else an even split in multiples of 64 rows
static inline __host__ __device__ int setup_pair_rows(int np, int ldz) {
    const int cap = ((48 * 1024 - 16 - PAIR_BLK * 8) / (ldz * 8)) & ~63;
    const int nch = (np + cap - 1) / cap;
    return ((np + nch - 1) / nch + 63) & ~63;
}
static inline __host__ __device__ size_t setup_pair_smem_bytes(int rows, int ldz) { return 16 + (size_t)PAIR_BLK * 8 + (size_t)rows * ldz * 8; }

// Forward stage 2, pair tasks: one CTA per (pair, row chunk, restart).  One TMA bulk copy each brings the pair block
// and the chunk's zeta rows (written by stage 1) into shared memory on one mbarrier; after that single wait no CTA-wide
// barrier.  Each warp sweeps octet pairs {2j, 2j+1}, j = warp, warp + 8, ..., the two octets as independent DMMA chains:
// first their B pieces, then their row operands.  Writes B_ab, U' (DMMA A fragments) and A' in the layout the tile kernels read.
#define SETUP_PAIR_WARPS 8
template <int DP>
__global__ void __launch_bounds__(32 * SETUP_PAIR_WARPS, 3) mm_setup2_pair_kernel(MMParams p, int rows) {
    PDL_ENTRY();
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int KS = DP / 4, NT = (DP + 7) / 8;
    constexpr int ldz = DP <= 4 ? 4 : (DP <= 12 ? 12 : 20);   // == L.ldz
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw);
    double* sblk = reinterpret_cast<double*>(smem_raw + 16);   // pair block (PAIR_*)
    double* sZ = sblk + PAIR_BLK;                              // zeta rows [c0, c0 + cm)
    const MMWs& L = p.L;
    const int n = p.gp.n, np = L.np;
    const int q = blockIdx.x, r = blockIdx.z, c0 = blockIdx.y * rows;
    const int cm = (np - c0) < rows ? (np - c0) : rows;        // multiple of 64
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    double* wsr = p.ws + (size_t)r * L.per_r;
    if (tid == 0) {
        mbar_init(bar, 1); mbar_fence_init();
        mbar_expect_tx(bar, (unsigned)(PAIR_BLK * 8 + cm * ldz * 8));
        tma_bulk_g2s(sblk, wsr + L.Qab + (size_t)q * PAIR_BLK, (unsigned)(PAIR_BLK * 8), bar);
        tma_bulk_g2s(sZ, wsr + L.zeta + (size_t)c0 * ldz, (unsigned)(cm * ldz * 8), bar);
    }
    __syncthreads();                                           // barrier initialisation visible to the waiting warps
    mbar_wait(bar, 0);
    double* Bq = wsr + L.Bq + (size_t)q * np + c0;
    double* Ar = wsr + L.Arow + (size_t)q * np + c0;
    double* uf = wsr + L.Ufrag + ((size_t)q * (np >> 3) + (c0 >> 3)) * (KS * 32);
    // two sweeps over the warp's octet pairs, so that only one sweep's pair constants are held in registers
    {
        double bqb[KS][NT];                                    // B fragments: B[k][n] = Qb[n][k]
#pragma unroll
        for (int ks = 0; ks < KS; ++ks)
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                const int i = 8 * nt + g;
                bqb[ks][nt] = i < DP ? sblk[PAIR_QB + i * DP + 4 * ks + t] : 0.0;
            }
        const double* pb = sblk + PAIR_PB;
        const double lsb = sblk[PAIR_SC + 2];
        for (int j = warp; 16 * j < cm; j += SETUP_PAIR_WARPS) {
            const double* const zr[2] = {sZ + (size_t)(16 * j + g) * ldz, sZ + (size_t)(16 * j + 8 + g) * ldz};
            const bool live[2] = {c0 + 16 * j + g < n, c0 + 16 * j + 8 + g < n};
            double bv[2];
            pair_b_octets<KS, 2>(bqb, pb, lsb, zr, live, lane, bv);
            if (t == 0) { Bq[16 * j + g] = bv[0]; Bq[16 * j + 8 + g] = bv[1]; }
        }
    }
    RowOpConsts<KS> roc;
    roc.load(sblk, lane);
    for (int j = warp; 16 * j < cm; j += SETUP_PAIR_WARPS) {
        const double* const zr[2] = {sZ + (size_t)(16 * j + g) * ldz, sZ + (size_t)(16 * j + 8 + g) * ldz};
        const bool live[2] = {c0 + 16 * j + g < n, c0 + 16 * j + 8 + g < n};
        double ua[2][KS], Apv[2];
        row_operands_octets<KS, 2>(roc, zr, live, lane, ua, Apv);
        if (t == 0) { Ar[16 * j + g] = Apv[0]; Ar[16 * j + 8 + g] = Apv[1]; }
#pragma unroll
        for (int o = 0; o < 2; ++o)
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) uf[(size_t)(2 * j + o) * (KS * 32) + ks * 32 + lane] = ua[o][ks];
    }
}

// both stages of one task in ONE launch -- stage 2 only consumes the stage-1 output of its own task,
// so warp 0 of the task's CTA runs the serial D x D part, a barrier publishes it (global writes of a CTA are
// visible to the CTA after __syncthreads), then all four warps sweep the centres.  One launch and one dependent
// kernel boundary less per moment match (two per rollout step with an RBF policy).
template <int DP, bool BWD>
__global__ void __launch_bounds__(128, 2) mm_setup_fused_kernel(MMParams p, int split) {
    PDL_ENTRY();
    // `split` CTAs share a pair task: each repeats the (short, serial) stage 1 -- they write identical pair blocks --
    // and sweeps every split-th 128-row chunk in stage 2, whose latency is what the single-restart step waits for
    const int r = blockIdx.y, E = p.gp.E;
    int task, part = 0, nparts = 1;
    if (!BWD && (int)blockIdx.x < E) task = blockIdx.x;                           // output task: one CTA (it reduces over all centres)
    else {
        const int k = BWD ? (int)blockIdx.x : (int)blockIdx.x - E;               // BWD: ordered pair tasks only
        task = E + k / split; part = k % split; nparts = split;
    }
    __shared__ double f_s[MAXD * SLD], f_L[MAXD * SLD], f_Q[MAXD * SLD], f_p[3][MAXD];
    setup_stage_s<DP>(p, r, f_s);
    __syncthreads();
    if (threadIdx.x < 32) mm_setup1_task<DP, BWD>(p, r, task, threadIdx.x, f_s, f_L, f_Q, f_p[0], f_p[1], f_p[2]);
    __syncthreads();
    mm_setup2_task<DP, BWD>(p, r, task, part, nparts);
    if (!BWD && blockIdx.x == 0) setup_publish_zeta<DP>(p, r, threadIdx.x, blockDim.x);   // forward: output task 0's CTA
}

// both stages
template <int DP, bool BWD>
static inline void mm_setup_launch(const MMParams& p, cudaStream_t st) {
    const int ntask = BWD ? p.L.P : p.gp.E + p.L.P;
    // ONE launch while the whole launch is small -- at most half the SMs' worth of CTAs: a single restart, or the RBF
    // policy's few tasks -- (latency regime: every launch on the serial path of a rollout step counts); anything bigger keeps
    // the two-stage form: stage 1 is register-hungry (218 registers at D = 12), fused it caps the occupancy of the throughput
    // stage, and in a sub-batch of a larger job its CTAs take SM slots from the other sub-batches' tile kernels.
    // PILCO_SETUP_FUSED=0/1 forces either (tuning switch).
    {
        static int mode = -1;
        if (mode < 0) { const char* e = getenv("PILCO_SETUP_FUSED"); mode = (e && (e[0] == '0' || e[0] == '1')) ? e[0] - '0' : 2; }
        const bool fused = mode == 2 ? mm_setup_is_fused(ntask, p.R, pilco_sm_count()) : mode == 1;
        if (fused) {
            // pair tasks are split over up to 3 CTAs, one 128-row chunk each (the stage-2 sweep is what the step waits for)
            int split = (p.L.np + 127) / 128;
            if (split > 3) split = 3;
            const int npair = p.L.P;                              // (BWD: P counts the ordered pairs)
            launch_hi(mm_setup_fused_kernel<DP, BWD>, dim3((ntask - npair) + npair * split, p.R), dim3(128), 0, st, p, split);
            return;
        }
    }
    launch_hi(mm_setup1_kernel<DP, BWD>, dim3((ntask + SETUP_WARPS - 1) / SETUP_WARPS + (BWD ? 0 : 1), p.R), dim3(32 * SETUP_WARPS), 0, st, p);
    if constexpr (BWD) {
        launch_hi(mm_setup2_bwd_kernel<DP>, dim3(ntask, p.R), dim3(128), 0, st, p);
    } else {
        const int rows = setup_pair_rows(p.L.np, p.L.ldz);
        launch_hi(mm_setup2_out_kernel<DP>, dim3(p.gp.E, p.R), dim3(128), 0, st, p);
        launch_hi(mm_setup2_pair_kernel<DP>, dim3(p.L.P, (p.L.np + rows - 1) / rows, p.R), dim3(32 * SETUP_PAIR_WARPS),
                  setup_pair_smem_bytes(rows, p.L.ldz), st, p, rows);
    }
}

// -------------------------------------------------------------------------------------------------
// tile kernel: CTA = (row blocks of 64 centres, pair, restart), 8 warps; a warp owns one row octet of each row block.
// The column operands (zeta [cols, ldz], B_q, beta_b) are staged in shared memory by TMA bulk copies; each warp
// sweeps all (valid) columns in groups of 4 DMMA tiles.  Off-diagonal pairs run mm_tile_body16 (two row blocks, i.e.
// 16 rows per warp, at a time -- below); diagonal pairs (a == b) run mm_tile_body and exploit the symmetry of
// G[n,m] L'[n,m]: only column tiles at or right of the row tile are visited, strictly-upper tiles count twice.
// -------------------------------------------------------------------------------------------------
static inline __host__ __device__ size_t mm_tile_smem_bytes(int np, int ldz) {
    const int cm = np < TILE_CM ? np : TILE_CM;
    return (size_t)cm * ldz * 8 + (size_t)cm * 16 + EXP_TAB_DOUBLES * 8 + 16;
}
// one partial per row octet (= per warp of a tile CTA): warps retire independently, no block reduction
static inline __host__ __device__ int mm_tile_slots(int np) { return np / 8; }

// Body of one tile CTA, specialised on the pair kind so that off-diagonal pairs carry neither the
// triangle bookkeeping nor the (predicated-off but still issued) trace FMAs of the diagonal pairs.
#ifdef PILCO_TILE_TIMING
// diagnostics build only (scripts/tile_phases.py): per CTA, warp 0 records clock64() at entry, after the row
// operands, after the first TMA wait, after the column sweep and at exit.
__device__ long long g_tile_timing[5 * 16384];
#define TILE_STAMP(k) do { if (threadIdx.x == 0) { const unsigned c_ = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z); \
                                                   if (c_ < 16384) g_tile_timing[5 * c_ + (k)] = clock64(); } } while (0)
#else
#define TILE_STAMP(k) do { } while (0)
#endif

template <int KS, bool SYM, bool DIAG>
__device__ __forceinline__ void mm_tile_body(const MMParams& p, int rpc) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    TILE_STAMP(0);
    const MMWs& L = p.L;
    constexpr int ldz = KS == 1 ? 4 : (KS <= 3 ? 12 : 20);    // == ldz_of(D) for every D with ksteps_of(D) == KS
    const int np = L.np, n = p.gp.n;
    const int CM = np < TILE_CM ? np : TILE_CM;
    double* sZ = reinterpret_cast<double*>(smem_raw);
    double* sBq = sZ + (size_t)CM * ldz;
    double* sBe = sBq + CM;
    double* tab = sBe + CM;
    uint64_t* bar = reinterpret_cast<uint64_t*>(tab + EXP_TAB_DOUBLES);

    // this CTA: pair q of restart r, row blocks [rb0, rb1) swept one after the other (the staged columns, the exp
    // table and the barrier are set up once per CTA; only the row operands change between passes)
    const int r = blockIdx.z, q = blockIdx.y;
    const int rb0 = blockIdx.x * rpc;
    const int rb1 = (rb0 + rpc) < L.NB ? (rb0 + rpc) : L.NB;
    int a, b;
    pair_decode(q, a, b);
    const double* wsr = p.ws + (size_t)r * L.per_r;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const double* ltab = EXP_LANE_TAB(tab, lane);      // this lane's copy of the exp table (conflict-free gather)
    const int ncol8 = (n + 7) & ~7;                    // columns at or beyond this are pure padding
    constexpr bool sympair = SYM;                      // symmetric pair (a == b): visit the upper triangle only
    constexpr bool diag = DIAG;                        // ... and (exact-GP mode) subtract the trace term
    const bool single = ncol8 <= CM;                   // one chunk holds every column: staged once for all passes

    if (tid == 0) { mbar_init(bar, 1); mbar_fence_init(); }

    // stage one column chunk (zeta rows, B_q, beta_b) and, with the first chunk, the exp table; symmetric pairs
    // skip everything left of the row tile `cfirst`
    auto issue_chunk = [&](int c0, int cfirst, bool with_table) {
        const int lo = cfirst > c0 ? cfirst - c0 : 0;                  // chunk-local first column (multiple of 64)
        const int cm = (np - c0) < CM ? (np - c0) : CM;
        const int ncopy = cm - lo;
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
        mbar_expect_tx(bar, (unsigned)(ncopy * ldz * 8 + ncopy * 16 + (with_table ? EXP_TAB_DOUBLES * 8 : 0)));
        tma_bulk_g2s(sZ + (size_t)lo * ldz, wsr + L.zeta + (size_t)(c0 + lo) * ldz, (unsigned)(ncopy * ldz * 8), bar);
        tma_bulk_g2s(sBq + lo, wsr + L.Bq + (size_t)q * np + c0 + lo, (unsigned)(ncopy * 8), bar);
        tma_bulk_g2s(sBe + lo, wsr + L.betap + (size_t)b * np + c0 + lo, (unsigned)(ncopy * 8), bar);
        if (with_table) tma_bulk_g2s(tab, g_exp_tab, (unsigned)(EXP_TAB_DOUBLES * 8), bar);
    };
    {
        const int cfirst0 = sympair ? rb0 * 64 : 0;
        const int cbeg0 = (cfirst0 / CM) * CM;
        if (tid == 0 && cbeg0 < ncol8) issue_chunk(cbeg0, cfirst0, true);
    }
    TILE_STAMP(1);
    __syncthreads();                                    // barrier initialisation visible to the waiting warps

    unsigned phase = 0;
    bool staged = true;                                 // the chunk issued at entry has not been consumed yet
    for (int rb = rb0; rb < rb1; ++rb) {
        const int row0 = rb * 64 + warp * 8;
        const int row = row0 + g;
        const bool active = row0 < n;                  // warp-uniform
        // row operands (materialised by setup stage 2): DMMA A fragments of U' and the scalar A'
        double ua[KS], Apv;
        {
            const double* uf = wsr + L.Ufrag + ((size_t)q * (np >> 3) + (row0 >> 3)) * (KS * 32);
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) ua[ks] = uf[ks * 32 + lane];
            Apv = wsr[L.Arow + (size_t)q * np + row];
        }
        // integer part of A' rides in the rounding constant of the exp, the fractional part scales the row sums
        double am, rowfac;
        exp_row_split(Apv, am, rowfac);
        const double ba = wsr[L.betap + (size_t)a * np + row] * rowfac;
        const double* ikrow = diag ? p.gp.iK + ((size_t)a * p.gp.ldk + row) * p.gp.ldk : nullptr;
        // first column this pass needs (symmetric pairs skip everything left of its row tile)
        const int cfirst = sympair ? rb * 64 : 0;
        const int cbeg = (cfirst / CM) * CM;

        double acc2 = 0.0, accd = 0.0, tr2 = 0.0, trd = 0.0;   // strictly-upper / diagonal-tile accumulators
        for (int c0 = cbeg; c0 < ncol8; c0 += CM) {
            const int lo = cfirst > c0 ? cfirst - c0 : 0;                  // chunk-local first column (multiple of 64)
            const int cm = (np - c0) < CM ? (np - c0) : CM;
            const int cend = (ncol8 - c0) < cm ? (ncol8 - c0) : cm;        // chunk-local end of valid columns
            if (staged) {                                                  // chunk issued at CTA entry
                mbar_wait(bar, phase);
                phase ^= 1;
                staged = false;
                TILE_STAMP(2);
            } else if (!single) {
                __syncthreads();                                           // all warps done with the previous chunk
                if (tid == 0) issue_chunk(c0, cfirst, false);
                mbar_wait(bar, phase);
                phase ^= 1;
            }
            if (active) {
                // symmetric pairs start at this warp's own row tile (global column row0)
                int cstart = lo;
                if (sympair && row0 > c0 + lo) cstart = (row0 - c0) & ~31;
                if (cstart < lo) cstart = lo;
                for (int cg = cstart; cg < cend; cg += 32) {
                    double2 ik[4];
                    if (diag) {
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            ik[j] = *reinterpret_cast<const double2*>(ikrow + c0 + cg + 8 * j + 2 * t);   // zero padded: always in bounds
                    }
                    // fast path: all four tiles valid and (symmetric pairs) strictly right of the diagonal tile
                    const bool full = (cg + 32 <= cend) && (!sympair || c0 + cg > row0);
                    if (full) {
                        double e[8];
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const double2 bq = *reinterpret_cast<const double2*>(sBq + cg + 8 * j + 2 * t);
                            e[2 * j] = bq.x; e[2 * j + 1] = bq.y;
                        }
#pragma unroll
                        for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                const double bf = sZ[(size_t)(cg + 8 * j + g) * ldz + 4 * ks + t];
                                dmma884(e[2 * j], e[2 * j + 1], ua[ks], bf);
                            }
                        }
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const double l0 = exp_shifted(e[2 * j], am, ltab), l1 = exp_shifted(e[2 * j + 1], am, ltab);
                            const double2 bb = *reinterpret_cast<const double2*>(sBe + cg + 8 * j + 2 * t);
                            acc2 = fma(bb.x, l0, acc2); acc2 = fma(bb.y, l1, acc2);
                            if (diag) { tr2 = fma(ik[j].x, l0, tr2); tr2 = fma(ik[j].y, l1, tr2); }
                        }
                        continue;
                    }
#pragma unroll 1
                    for (int j = 0; j < 4; ++j) {
                        const int col = cg + 8 * j;
                        const int gcol = c0 + col;
                        if (col < cend && (!sympair || gcol >= row0)) {         // warp-uniform
                            const double2 bq = *reinterpret_cast<const double2*>(sBq + col + 2 * t);
                            double e0 = bq.x, e1 = bq.y;
#pragma unroll
                            for (int ks = 0; ks < KS; ++ks) {
                                const double bf = sZ[(size_t)(col + g) * ldz + 4 * ks + t];
                                dmma884(e0, e1, ua[ks], bf);
                            }
                            const double l0 = exp_shifted(e0, am, ltab), l1 = exp_shifted(e1, am, ltab);
                            const double2 bb = *reinterpret_cast<const double2*>(sBe + col + 2 * t);
                            const double2 ikj = diag ? *reinterpret_cast<const double2*>(ikrow + gcol + 2 * t) : make_double2(0.0, 0.0);
                            if (sympair && gcol == row0) {
                                accd = fma(bb.x, l0, accd); accd = fma(bb.y, l1, accd);
                                trd = fma(ikj.x, l0, trd); trd = fma(ikj.y, l1, trd);
                            } else {
                                acc2 = fma(bb.x, l0, acc2); acc2 = fma(bb.y, l1, acc2);
                                tr2 = fma(ikj.x, l0, tr2); tr2 = fma(ikj.y, l1, tr2);
                            }
                        }
                    }
                }
            }
        }
        if (rb + 1 == rb1) TILE_STAMP(3);
        // row sums -> beta_a-weighted total; symmetric pairs: diagonal tile once, strictly-upper tiles twice
        double acc = sympair ? accd + 2.0 * acc2 : acc2;
        double tr = sympair ? trd + 2.0 * tr2 : tr2;
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
        double v = (t == 0) ? ba * acc : 0.0;
        if (diag) v = fma(-tr, rowfac, v);                  // trace term (per-lane partial), same warp reduction
        v = warp_sum(v);
        if (lane == 0)
            p.ws[(size_t)r * L.per_r + L.Tpart + (size_t)q * mm_tile_slots(np) + rb * 8 + warp] = active ? v : 0.0;
    }
    TILE_STAMP(4);
}

// -------------------------------------------------------------------------------------------------
// Off-diagonal pairs with TWO row octets per warp (the 2 CTAs/SM instantiation): the warp takes its octet of two
// consecutive row blocks at a time, so every column operand it reads from shared memory -- the DMMA B fragments of
// zeta, B_q, beta_b -- feeds two tiles instead of one: 36 instead of 56 LDS per 8 tiles, and twice the independent
// DMMA -> exp chains in flight per warp (scripts/ubench/fp64_mix.cu, `full16` against `full`, times the instruction
// mix alone).  An odd last row
// block runs the one-octet form of the same code.  Every group is fully unrolled (1-4 column tiles): no per-tile
// branches anywhere.  Same staging (TMA bulk copies on one mbarrier), same per-octet outputs (Tpart) as mm_tile_body.
// -------------------------------------------------------------------------------------------------
template <int KS, int NR>
__device__ __forceinline__ void tile_sweep16(const double* __restrict__ sZ, const double* __restrict__ sBq,
                                             const double* __restrict__ sBe, const double* __restrict__ ltab, int cend,
                                             const double (&ua)[2][KS], const double (&am)[2], double (&acc)[2], int g, int t) {
    constexpr int ldz = KS == 1 ? 4 : (KS <= 3 ? 12 : 20);
    int cg = 0;
    auto group = [&](auto nt_c) {
        constexpr int NTL = decltype(nt_c)::value;
        double e[NR][2 * NTL];
#pragma unroll
        for (int j = 0; j < NTL; ++j) {
            const double2 bq = *reinterpret_cast<const double2*>(sBq + cg + 8 * j + 2 * t);
#pragma unroll
            for (int o = 0; o < NR; ++o) { e[o][2 * j] = bq.x; e[o][2 * j + 1] = bq.y; }
        }
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
            for (int j = 0; j < NTL; ++j) {
                const double bf = sZ[(size_t)(cg + 8 * j + g) * ldz + 4 * ks + t];
#pragma unroll
                for (int o = 0; o < NR; ++o) dmma884(e[o][2 * j], e[o][2 * j + 1], ua[o][ks], bf);
            }
        }
#pragma unroll
        for (int j = 0; j < NTL; ++j) {
            const double2 bb = *reinterpret_cast<const double2*>(sBe + cg + 8 * j + 2 * t);
#pragma unroll
            for (int o = 0; o < NR; ++o) {
                const double l0 = exp_shifted(e[o][2 * j], am[o], ltab), l1 = exp_shifted(e[o][2 * j + 1], am[o], ltab);
                acc[o] = fma(bb.x, l0, acc[o]); acc[o] = fma(bb.y, l1, acc[o]);
            }
        }
    };
    for (; cg + 32 <= cend; cg += 32) group(std::integral_constant<int, 4>{});
    const int ntl = (cend - cg) >> 3;                                   // 0 .. 3 tiles left (cend is a multiple of 8)
    if (ntl == 3) group(std::integral_constant<int, 3>{});
    else if (ntl == 2) group(std::integral_constant<int, 2>{});
    else if (ntl == 1) group(std::integral_constant<int, 1>{});
}

template <int KS>
__device__ __forceinline__ void mm_tile_body16(const MMParams& p, int rpc) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    TILE_STAMP(0);
    const MMWs& L = p.L;
    constexpr int ldz = KS == 1 ? 4 : (KS <= 3 ? 12 : 20);
    const int np = L.np, n = p.gp.n;
    const int CM = np < TILE_CM ? np : TILE_CM;
    double* sZ = reinterpret_cast<double*>(smem_raw);
    double* sBq = sZ + (size_t)CM * ldz;
    double* sBe = sBq + CM;
    double* tab = sBe + CM;
    uint64_t* bar = reinterpret_cast<uint64_t*>(tab + EXP_TAB_DOUBLES);

    const int r = blockIdx.z, q = blockIdx.y;
    const int rb0 = blockIdx.x * rpc;
    const int rb1 = (rb0 + rpc) < L.NB ? (rb0 + rpc) : L.NB;
    int a, b;
    pair_decode(q, a, b);
    const double* wsr = p.ws + (size_t)r * L.per_r;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const double* ltab = EXP_LANE_TAB(tab, lane);
    const int ncol8 = (n + 7) & ~7;
    const bool single = ncol8 <= CM;

    if (tid == 0) { mbar_init(bar, 1); mbar_fence_init(); }
    auto issue_chunk = [&](int c0, bool with_table) {
        const int cm = (np - c0) < CM ? (np - c0) : CM;
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
        mbar_expect_tx(bar, (unsigned)(cm * ldz * 8 + cm * 16 + (with_table ? EXP_TAB_DOUBLES * 8 : 0)));
        tma_bulk_g2s(sZ, wsr + L.zeta + (size_t)c0 * ldz, (unsigned)(cm * ldz * 8), bar);
        tma_bulk_g2s(sBq, wsr + L.Bq + (size_t)q * np + c0, (unsigned)(cm * 8), bar);
        tma_bulk_g2s(sBe, wsr + L.betap + (size_t)b * np + c0, (unsigned)(cm * 8), bar);
        if (with_table) tma_bulk_g2s(tab, g_exp_tab, (unsigned)(EXP_TAB_DOUBLES * 8), bar);
    };
    if (tid == 0) issue_chunk(0, true);
    TILE_STAMP(1);
    __syncthreads();                                    // barrier initialisation visible to the waiting warps

    unsigned phase = 0;
    bool staged = true;                                 // the chunk issued at entry has not been consumed yet
    for (int rb = rb0; rb < rb1; rb += 2) {
        const int nr = rb + 1 < rb1 ? 2 : 1;            // row blocks of this pass (uniform over the CTA)
        int row0[2];
        bool act[2];
        double ua[2][KS], am[2], ba[2], acc[2];
#pragma unroll
        for (int o = 0; o < 2; ++o) {
            row0[o] = (rb + o) * 64 + warp * 8;
            act[o] = o < nr && row0[o] < n;             // warp-uniform; act[1] implies act[0]
            am[o] = EXP_MAGIC; ba[o] = 0.0; acc[o] = 0.0;
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) ua[o][ks] = 0.0;
            if (o < nr) {
                // row operands (materialised by setup stage 2): DMMA A fragments of U' and the scalar A', whose integer
                // part rides in the rounding constant of the exp while the fractional part scales the row sums
                const int row = row0[o] + g;
                const double* uf = wsr + L.Ufrag + ((size_t)q * (np >> 3) + (row0[o] >> 3)) * (KS * 32);
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) ua[o][ks] = uf[ks * 32 + lane];
                double rowfac;
                exp_row_split(wsr[L.Arow + (size_t)q * np + row], am[o], rowfac);
                ba[o] = wsr[L.betap + (size_t)a * np + row] * rowfac;
            }
        }
        for (int c0 = 0; c0 < ncol8; c0 += CM) {
            const int cm = (np - c0) < CM ? (np - c0) : CM;
            const int cend = (ncol8 - c0) < cm ? (ncol8 - c0) : cm;        // chunk-local end of valid columns
            if (staged) {                                                  // chunk issued at CTA entry
                mbar_wait(bar, phase);
                phase ^= 1;
                staged = false;
                TILE_STAMP(2);
            } else if (!single) {
                __syncthreads();                                           // all warps done with the previous chunk
                if (tid == 0) issue_chunk(c0, false);
                mbar_wait(bar, phase);
                phase ^= 1;
            }
            if (act[1]) tile_sweep16<KS, 2>(sZ, sBq, sBe, ltab, cend, ua, am, acc, g, t);
            else if (act[0]) tile_sweep16<KS, 1>(sZ, sBq, sBe, ltab, cend, ua, am, acc, g, t);
        }
        if (rb + 2 >= rb1) TILE_STAMP(3);
        // row sums -> beta_a-weighted totals, one partial per row octet
#pragma unroll
        for (int o = 0; o < 2; ++o) {
            if (o < nr) {
                double s = acc[o];
                s += __shfl_xor_sync(0xffffffffu, s, 1);
                s += __shfl_xor_sync(0xffffffffu, s, 2);
                double v = (t == 0) ? ba[o] * s : 0.0;
                v = warp_sum(v);
                if (lane == 0)
                    p.ws[(size_t)r * L.per_r + L.Tpart + (size_t)q * mm_tile_slots(np) + (rb + o) * 8 + warp] = act[o] ? v : 0.0;
            }
        }
    }
    TILE_STAMP(4);
}

// rpc = row blocks per CTA (launch_tile chooses it: all of them once the grid still covers the SMs)
template <int KS, int MINB, bool TWO = (MINB == 2)>
__global__ void __launch_bounds__(256, MINB) mm_tile_kernel(MMParams p, int rpc) {
    PDL_ENTRY();
    int a, b;
    pair_decode(blockIdx.y, a, b);
    if (a != b) {
        if (TWO) mm_tile_body16<KS>(p, rpc);                // two row octets per warp (the default instantiation)
        else mm_tile_body<KS, false, false>(p, rpc);
    }
    else if (p.gp.mode == 0 && p.gp.iK != nullptr) mm_tile_body<KS, true, true>(p, rpc);
    else mm_tile_body<KS, true, false>(p, rpc);
}

// -------------------------------------------------------------------------------------------------
// Off-diagonal pairs on Hopper's native 16x8 MMA shapes.  The two row octets of mm_tile_body16 share every B fragment,
// so their two 8x8 exponent tiles are ONE 16x8 tile: A = the two octets' U' fragments (rows g and g + 8), C = the two
// octets' C fragments side by side, K = DP in one MMA per K chunk (mma16_k) instead of 2 KS DMMA.8x8x4.  Same staging,
// same exp and weighted sums, same per-octet outputs (Tpart) as mm_tile_body16.
// A pass with ONE row block left (an odd last block) keeps the 16-row shape too: warps 0-3 take the octet pairs
// {2w, 2w + 1} of that block over all columns, warps 4-7 have no rows in that pass (the other CTAs on the SM use the
// pipe).  An octet's sum is the same whichever pass form it ran in -- the row blocks per CTA, and with them the odd
// blocks, follow the batch size, and a restart's result must not.
// -------------------------------------------------------------------------------------------------
template <int KS>
__device__ __forceinline__ void tile_sweep_m16(const double* __restrict__ sZ, const double* __restrict__ sBq,
                                               const double* __restrict__ sBe, const double* __restrict__ ltab, int cbeg, int cend,
                                               const double (&af)[2 * KS], const double (&am)[2], double (&acc)[2], int g, int t) {
    constexpr int ldz = KS == 1 ? 4 : (KS <= 3 ? 12 : 20);
    int cg = cbeg;
    auto group = [&](auto nt_c) {
        constexpr int NTL = decltype(nt_c)::value;
        double e[NTL][4];
#pragma unroll
        for (int j = 0; j < NTL; ++j) {
            const double2 bq = *reinterpret_cast<const double2*>(sBq + cg + 8 * j + 2 * t);
            e[j][0] = bq.x; e[j][1] = bq.y; e[j][2] = bq.x; e[j][3] = bq.y;
        }
#pragma unroll
        for (int j = 0; j < NTL; ++j) {
            double bf[KS];
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) bf[ks] = sZ[(size_t)(cg + 8 * j + g) * ldz + 4 * ks + t];
            mma16_k<KS>(e[j], af, bf);
        }
#pragma unroll
        for (int j = 0; j < NTL; ++j) {
            const double2 bb = *reinterpret_cast<const double2*>(sBe + cg + 8 * j + 2 * t);
#pragma unroll
            for (int o = 0; o < 2; ++o) {
                const double l0 = exp_shifted(e[j][2 * o], am[o], ltab), l1 = exp_shifted(e[j][2 * o + 1], am[o], ltab);
                acc[o] = fma(bb.x, l0, acc[o]); acc[o] = fma(bb.y, l1, acc[o]);
            }
        }
    };
    // groups of 4 column tiles (KS = 3: 3, KS = 4: 2 -- with the wider A fragments larger groups spill at 80 registers)
    constexpr int GM = KS == 4 ? 2 : (KS == 3 ? 3 : 4);
    for (; cg + 8 * GM <= cend; cg += 8 * GM) group(std::integral_constant<int, GM>{});
    const int ntl = (cend - cg) >> 3;                                   // 0 .. GM - 1 tiles left (cend - cbeg is a multiple of 8)
    if (GM == 4 && ntl == 3) group(std::integral_constant<int, 3>{});
    else if (ntl == 2) group(std::integral_constant<int, 2>{});
    else if (ntl == 1) group(std::integral_constant<int, 1>{});
}

template <int KS>
__device__ __forceinline__ void mm_tile_body_m16(const MMParams& p, int rpc) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    TILE_STAMP(0);
    const MMWs& L = p.L;
    constexpr int ldz = KS == 1 ? 4 : (KS <= 3 ? 12 : 20);
    const int np = L.np, n = p.gp.n;
    const int CM = np < TILE_CM ? np : TILE_CM;
    double* sZ = reinterpret_cast<double*>(smem_raw);
    double* sBq = sZ + (size_t)CM * ldz;
    double* sBe = sBq + CM;
    double* tab = sBe + CM;
    uint64_t* bar = reinterpret_cast<uint64_t*>(tab + EXP_TAB_DOUBLES);

    const int r = blockIdx.z, q = blockIdx.y;
    const int rb0 = blockIdx.x * rpc;
    const int rb1 = (rb0 + rpc) < L.NB ? (rb0 + rpc) : L.NB;
    int a, b;
    pair_decode(q, a, b);
    const double* wsr = p.ws + (size_t)r * L.per_r;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const double* ltab = EXP_LANE_TAB(tab, lane);
    const int ncol8 = (n + 7) & ~7;
    const bool single = ncol8 <= CM;

    if (tid == 0) { mbar_init(bar, 1); mbar_fence_init(); }
    auto issue_chunk = [&](int c0, bool with_table) {
        const int cm = (np - c0) < CM ? (np - c0) : CM;
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
        mbar_expect_tx(bar, (unsigned)(cm * ldz * 8 + cm * 16 + (with_table ? EXP_TAB_DOUBLES * 8 : 0)));
        tma_bulk_g2s(sZ, wsr + L.zeta + (size_t)c0 * ldz, (unsigned)(cm * ldz * 8), bar);
        tma_bulk_g2s(sBq, wsr + L.Bq + (size_t)q * np + c0, (unsigned)(cm * 8), bar);
        tma_bulk_g2s(sBe, wsr + L.betap + (size_t)b * np + c0, (unsigned)(cm * 8), bar);
        if (with_table) tma_bulk_g2s(tab, g_exp_tab, (unsigned)(EXP_TAB_DOUBLES * 8), bar);
    };
    if (tid == 0) issue_chunk(0, true);
    TILE_STAMP(1);
    __syncthreads();                                    // barrier initialisation visible to the waiting warps

    unsigned phase = 0;
    bool staged = true;                                 // the chunk issued at entry has not been consumed yet
    for (int rb = rb0; rb < rb1; rb += 2) {
        const bool odd = rb + 1 >= rb1;                 // one row block left (uniform over the CTA)
        // this warp's two octets (global octet indices): octet w of both row blocks, or octets 2w, 2w + 1 of the odd block
        const int oct0 = odd ? rb * 8 + 2 * (warp & 3) : rb * 8 + warp;
        const int ostep = odd ? 1 : 8;
        const bool mine = !odd || warp < 4;             // warp-uniform: does this warp own rows in this pass
        int row0[2];
        bool act[2];
        double af[2 * KS], am[2], ba[2], acc[2];
#pragma unroll
        for (int o = 0; o < 2; ++o) {
            row0[o] = 8 * (oct0 + o * ostep);
            act[o] = mine && row0[o] < n;               // warp-uniform; act[1] implies act[0]
            am[o] = EXP_MAGIC; ba[o] = 0.0; acc[o] = 0.0;
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) af[2 * ks + o] = 0.0;
            if (act[o]) {
                // row operands (materialised by setup stage 2): U' fragments of the octet as rows 8o + g of the 16x8 A
                // operand, and the scalar A' (integer part -> exp rounding constant, fractional part -> row factor)
                const int row = row0[o] + g;
                const double* uf = wsr + L.Ufrag + ((size_t)q * (np >> 3) + (row0[o] >> 3)) * (KS * 32);
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) af[2 * ks + o] = uf[ks * 32 + lane];
                double rowfac;
                exp_row_split(wsr[L.Arow + (size_t)q * np + row], am[o], rowfac);
                ba[o] = wsr[L.betap + (size_t)a * np + row] * rowfac;
            }
        }
        for (int c0 = 0; c0 < ncol8; c0 += CM) {
            const int cm = (np - c0) < CM ? (np - c0) : CM;
            const int cend = (ncol8 - c0) < cm ? (ncol8 - c0) : cm;        // chunk-local end of valid columns
            if (staged) {                                                  // chunk issued at CTA entry
                mbar_wait(bar, phase);
                phase ^= 1;
                staged = false;
                TILE_STAMP(2);
            } else if (!single) {
                __syncthreads();                                           // all warps done with the previous chunk
                if (tid == 0) issue_chunk(c0, false);
                mbar_wait(bar, phase);
                phase ^= 1;
            }
            if (act[0]) tile_sweep_m16<KS>(sZ, sBq, sBe, ltab, 0, cend, af, am, acc, g, t);
        }
        if (rb + 2 >= rb1) TILE_STAMP(3);
        // row sums -> beta_a-weighted totals, one partial per row octet
        double* Tp = p.ws + (size_t)r * L.per_r + L.Tpart + (size_t)q * mm_tile_slots(np);
        double v[2];
#pragma unroll
        for (int o = 0; o < 2; ++o) {
            double s = acc[o];
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            v[o] = warp_sum((t == 0) ? ba[o] * s : 0.0);
        }
        if (mine && lane == 0) {
            Tp[oct0] = act[0] ? v[0] : 0.0;
            Tp[oct0 + ostep] = act[1] ? v[1] : 0.0;
        }
    }
    TILE_STAMP(4);
}

// 3 CTAs/SM (<= 80 registers); diagonal pairs keep the one-octet 8x8x4 body (triangle + trace bookkeeping)
template <int KS>
__global__ void __launch_bounds__(256, 3) mm_tile_m16_kernel(MMParams p, int rpc) {
    PDL_ENTRY();
    int a, b;
    pair_decode(blockIdx.y, a, b);
    if (a != b) mm_tile_body_m16<KS>(p, rpc);
    else if (p.gp.mode == 0 && p.gp.iK != nullptr) mm_tile_body<KS, true, true>(p, rpc);
    else mm_tile_body<KS, true, false>(p, rpc);
}

// -------------------------------------------------------------------------------------------------
// finish
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mm_finish_device(const MMParams& p, int r) {
    const pilco_gp_model& gp = p.gp;
    const int E = gp.E;
    const MMWs& L = p.L;
    const double* wsr = p.ws + (size_t)r * L.per_r;
    const double* sf2 = gp.sf2 + (size_t)r * gp.sf2_bs;
    // two adjacent lanes per pair: each sums every second per-row-octet partial (independent loads the compiler
    // pipelines), one shuffle combines them -- this sits on the serial path of every rollout step.  Fixed order:
    // deterministic.
    const int slots = mm_tile_slots(L.np);
    const int half = threadIdx.x & 1, per_round = blockDim.x >> 1;
    for (int base = 0; base < L.P; base += per_round) {      // uniform trip count: the shuffle below is warp-wide
        const int q = base + (threadIdx.x >> 1);
        const bool valid = q < L.P;
        double T = 0.0;
        if (valid)
            for (int k = half; k < slots; k += 2) T += wsr[L.Tpart + (size_t)q * slots + k];
        T += __shfl_xor_sync(0xffffffffu, T, 1);
        if (valid && half == 0) {
            int a, b;
            pair_decode(q, a, b);
            const double Ma = p.M[(size_t)r * E + a], Mb = p.M[(size_t)r * E + b];
            double v = T - Ma * Mb;
            if (a == b) v += (gp.mode == 0) ? sf2[a] : 1e-6;
            p.S[((size_t)r * E + a) * E + b] = v;
            p.S[((size_t)r * E + b) * E + a] = v;
        }
    }
}

static __global__ void __launch_bounds__(128) mm_finish_kernel(MMParams p) {
    PDL_ENTRY();
    mm_finish_device(p, blockIdx.x);
}

#endif  // __CUDACC__

// host-side launcher shared by mm_forward.cu and rollout.cu: setup, tile (taped when p.tape), finish (with_finish).
// ev: null, or 4 events recorded before the setup, the tile pass and the finish and after the finish.
int mm_forward_launch(const MMParams& p, cudaStream_t st, bool with_finish, cudaEvent_t* ev = nullptr);
int mm_check_model(const pilco_gp_model* gp);
