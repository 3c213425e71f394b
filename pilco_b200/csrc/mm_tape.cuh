// mm_tape.cuh -- "taped" moment match: the forward tile pass that also leaves what the reverse sweep needs.
//
// The reference differentiates MGPR.predict_given_factorizations (pilco/models/mgpr.py:91-149) with TensorFlow
// autodiff, which keeps every [E,E,N,N] intermediate of every rollout step.  The dynamics GP's inputs X are
// constants of the policy objective (pilco/models/pilco.py:80-82 freezes the model), so its VJP needs only the
// cotangents of the input moments (m, s) -- and those depend on the N x N matrix H_ab = G_ab o L'_ab of a pair only
// through its row sums, its column sums and the ONE product H_ab Z  (Z = centred inputs, N x D):
//     d T_ab / dQ       = Za' diag(hr) Za + Zb' diag(hc) Zb + Za' (H Z) Pb + (Za' (H Z) Pb)'      (Za = Z diag p_a)
//     d T_ab / dm       = -(sum_n hr_n d e/d zeta_n + sum_m hc_m d e/d zeta_m)                      (linear in hr, hc)
//     d T_ab / dlogdetR = -T_ab / 2
// These are linear in the (not yet known) cotangent of S_ab, so the FORWARD tile pass can produce them unweighted
// while it has L' in registers: per 8x8 tile two/four extra DMMA (H Z) next to the exponent's KS DMMA and the exp.
// The reverse sweep of the dynamics GP then never recomputes an exponential: it is a few small (D x N)(N x D)
// products per pair (mm_tape_bfinish_kernel).  Forward + backward cost ~1.9 tile passes instead of 1 + 4.
//
// Tape of one moment-match call, per restart (doubles): Q[P,D,D], C[P,D,D] = (s + diag 1/delta)^-1, logdetR[P],
// hr[P,np], hc[P,cs,np] (cs = row splits of a pair over CTAs), HZ[P,np,ldh].
#pragma once
#include "mm_kernels.cuh"

// row splits of one pair over CTAs: 1 once pairs x restarts fill the machine twice over
// (host only: depends on the current device's SM count.  A tape lives in one device's memory and its forward pass and
// reverse sweep run on that device, so both derive the same layout; every entry point also checks tape_bytes against the
// layout of the current device, so a tape sized on a device with fewer splits is rejected, never overrun.)
static inline int mm_tape_splits(int n, int P, int R) { return mm_tape_splits_on(n, P, R, pilco_sm_count()); }

static inline MMTapeL mm_tape_layout(int n, int D, int E, int R) {
    MMTapeL T;
    T.np = pad64(n); T.P = npairs_of(E);
    T.ldh = ldz_of(D);            // row stride of HZ: 4 / 12 / 20, bank-conflict free as a DMMA B operand (like zeta)
    T.cs = mm_tape_splits(n, T.P, R);
    size_t o = 0;
    auto take = [&](size_t len) { size_t at = o; o += (len + 1) & ~(size_t)1; return at; };
    T.Q = take((size_t)T.P * D * D);
    T.C = take((size_t)T.P * D * D);
    T.Ld = take(T.P);
    T.hr = take((size_t)T.P * T.np);
    T.hc = take((size_t)T.P * T.cs * T.np);
    T.HZ = take((size_t)T.P * T.np * T.ldh);
    T.per_r = o;
    return T;
}

#define TAPE_MAX_NP 2048        // per-warp column sums live in shared memory: 8 warps x np doubles

static inline __host__ __device__ size_t mm_tape_smem_bytes(int np, int ldz) {
    const int cm = np < TILE_CM ? np : TILE_CM;
    return (size_t)cm * ldz * 8 + (size_t)cm * 16 + EXP_TAB_DOUBLES * 8 + 16 + (size_t)8 * np * 8;
}

#ifdef __CUDACC__

// One column sweep of NR (1 or 2) row octets of one warp over the staged columns [cbeg, cend) of a chunk.
//   exponent tile  e = B[m] + U'[n].zeta_m  by KS DMMA; its B fragment takes the centres in the order
//   pi = (0,4,1,5,2,6,3,7), so the C fragment of lane (g,t) holds columns (t, 4+t) of row g -- which IS the A
//   fragment layout of the second product (k-step 0: column t, k-step 1: column 4+t): no shuffles in between.
//   w = G o L' (without the row factor rf);  row sums hl;  column partials sum_o rf_o w (butterfly over the 8 rows);
//   HZ += w . zeta[cols]  by 2 NT DMMA.
template <int KS, bool DIAG, int NR>
__device__ __forceinline__ void tape_sweep(const double* __restrict__ sZ, const double* __restrict__ sBq,
                                           const double* __restrict__ sBe, const double* __restrict__ tab,
                                           int cbeg, int cend, int c0,
                                           const double (&ua)[2][KS], const double (&am)[2], const double (&rf)[2],
                                           const double (&bn)[2], const double* const (&ikrow)[2],
                                           double (&hl)[2], double (&hz)[2][(4 * KS + 7) / 8][2],
                                           double* __restrict__ sCsw, int lane) {
    constexpr int ldz = KS == 1 ? 4 : (KS <= 3 ? 12 : 20);
    constexpr int NT = (4 * KS + 7) / 8;
    constexpr bool ONES = (KS & 1) != 0;                       // DP = 4 KS = 4 (mod 8)
    const int g = lane >> 2, t = lane & 3;
    const int pg = (g >> 1) | ((g & 1) << 2);                  // pi(g)
    const double* ltab = EXP_LANE_TAB(tab, lane);
    for (int cg = cbeg; cg < cend; cg += 8) {
        const double bq0 = sBq[cg + t], bq1 = sBq[cg + 4 + t];
        const double bb0 = sBe[cg + t], bb1 = sBe[cg + 4 + t];
        double bf[KS];
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) bf[ks] = sZ[(size_t)(cg + pg) * ldz + 4 * ks + t];
        double zb[2][NT];
#pragma unroll
        for (int k2 = 0; k2 < 2; ++k2)
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) zb[k2][nt] = sZ[(size_t)(cg + 4 * k2 + t) * ldz + 8 * nt + g];
        // DP = 4 (mod 8): column DP of the last n-tile is free -- a column of ones there makes the second product
        // deliver the row sums as HZ[:, DP] (lanes t == 2, element 0) and saves the explicit adds
        if (ONES && g == 4) { zb[0][NT - 1] = 1.0; zb[1][NT - 1] = 1.0; }
        double cs0 = 0.0, cs1 = 0.0;
#pragma unroll
        for (int j = 0; j < NR; ++j) {
            double e0 = bq0, e1 = bq1;
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) dmma884(e0, e1, ua[j][ks], bf[ks]);
            const double l0 = exp_shifted(e0, am[j], ltab), l1 = exp_shifted(e1, am[j], ltab);
            double w0, w1;
            if (DIAG) {
                const double ik0 = ikrow[j][c0 + cg + t], ik1 = ikrow[j][c0 + cg + 4 + t];   // zero padded: in bounds
                w0 = fma(bn[j], bb0, -ik0) * l0;
                w1 = fma(bn[j], bb1, -ik1) * l1;
            } else {
                w0 = bb0 * l0; w1 = bb1 * l1;
            }
            if (!ONES) hl[j] += w0 + w1;
            if (!DIAG) { cs0 = fma(rf[j], w0, cs0); cs1 = fma(rf[j], w1, cs1); }
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                dmma884(hz[j][nt][0], hz[j][nt][1], w0, zb[0][nt]);
                dmma884(hz[j][nt][0], hz[j][nt][1], w1, zb[1][nt]);
            }
        }
        // column sums of this 8-column tile over the warp's rows: butterfly over g, lanes g == 0 own the result.
        // Diagonal pairs of an exact GP skip them: H = G o L' is symmetric there, so hc = hr (the finish task reads hr)
        if (!DIAG) {
            // reduce-scatter: the first exchange (rows g <-> g ^ 4) hands each lane the partner's partial of ONE of its two
            // columns (g < 4 keeps column t, g >= 4 keeps column 4 + t), so the remaining two levels move one value, not
            // two: 3 instead of 6 64-bit shuffles per tile (the shuffles, not the adds, are what this costs)
            const bool up = (g & 4) != 0;
            double keep = up ? cs1 : cs0;
            const double send = up ? cs0 : cs1;
            keep += __shfl_xor_sync(0xffffffffu, send, 16);
            keep += __shfl_xor_sync(0xffffffffu, keep, 8);
            keep += __shfl_xor_sync(0xffffffffu, keep, 4);
            if ((g & 3) == 0) sCsw[c0 + cg + (up ? 4 : 0) + t] += keep;
        }
    }
}

// CTA = (row split, pair, restart); 8 warps; warp gw of the pair takes the row octets gw, gw + GW, ... two at a time.
template <int KS, bool DIAG>
__device__ __forceinline__ void mm_tape_body(const MMParams& p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int ldz = KS == 1 ? 4 : (KS <= 3 ? 12 : 20);
    constexpr int NT = (4 * KS + 7) / 8;
    const MMWs& L = p.L;
    const MMTapeL& TL = p.TL;
    const int np = L.np, n = p.gp.n;
    const int CM = np < TILE_CM ? np : TILE_CM;
    double* sZ = reinterpret_cast<double*>(smem_raw);
    double* sBq = sZ + (size_t)CM * ldz;
    double* sBe = sBq + CM;
    double* tab = sBe + CM;
    uint64_t* bar = reinterpret_cast<uint64_t*>(tab + EXP_TAB_DOUBLES);
    double* sCs = reinterpret_cast<double*>(bar + 2);          // [8 warps][np] column-sum partials

    const int r = blockIdx.z, q = blockIdx.y, sidx = blockIdx.x, cs = gridDim.x;
    int a, b;
    pair_decode(q, a, b);
    const double* wsr = p.ws + (size_t)r * L.per_r;
    double* tpr = p.tape + (size_t)r * TL.per_r;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int NO = (n + 7) >> 3, NS = np >> 3;                 // live row octets / partial-sum slots of a pair
    const int ncol8 = (n + 7) & ~7;
    const bool single = ncol8 <= CM;
    double* sCsw = sCs + (size_t)warp * np;

    if (tid == 0) { mbar_init(bar, 1); mbar_fence_init(); }
    for (int c = lane; c < np; c += 32) sCsw[c] = 0.0;
    auto issue_chunk = [&](int c0, bool with_table) {
        const int cm = (np - c0) < CM ? (np - c0) : CM;
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
        mbar_expect_tx(bar, (unsigned)(cm * ldz * 8 + cm * 16 + (with_table ? EXP_TAB_DOUBLES * 8 : 0)));
        tma_bulk_g2s(sZ, wsr + L.zeta + (size_t)c0 * ldz, (unsigned)(cm * ldz * 8), bar);
        tma_bulk_g2s(sBq, wsr + L.Bq + (size_t)q * np + c0, (unsigned)(cm * 8), bar);
        tma_bulk_g2s(sBe, wsr + L.betap + (size_t)b * np + c0, (unsigned)(cm * 8), bar);
        if (with_table) tma_bulk_g2s(tab, g_exp_tab, (unsigned)(EXP_TAB_DOUBLES * 8), bar);
    };
    __syncthreads();                                    // barrier initialised before the first arrive / wait
    if (tid == 0) issue_chunk(0, true);

    const int GW = cs * 8, gw = sidx * 8 + warp;
    const int npass = (NS + 2 * GW - 1) / (2 * GW);     // uniform over the CTA (barriers inside when !single)
    unsigned phase = 0;
    bool staged = true;
    for (int pass = 0; pass < npass; ++pass) {
        int oct[2];
        oct[0] = gw + (2 * pass) * GW; oct[1] = gw + (2 * pass + 1) * GW;
        const int nlive = (oct[0] < NO) + (oct[1] < NO);       // warp-uniform; oct[0] < oct[1]
        double ua[2][KS], am[2], rf[2], bn[2], hl[2], hz[2][NT][2];
        const double* ikrow[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            hl[j] = 0.0; bn[j] = 0.0; rf[j] = 0.0; am[j] = EXP_MAGIC; ikrow[j] = nullptr;
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) { hz[j][nt][0] = hz[j][nt][1] = 0.0; }
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) ua[j][ks] = 0.0;
            if (oct[j] < NO) {
                const int row = 8 * oct[j] + g;
                const double* uf = wsr + L.Ufrag + ((size_t)q * NS + oct[j]) * (KS * 32);
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) ua[j][ks] = uf[ks * 32 + lane];
                double rowfac;
                exp_row_split(wsr[L.Arow + (size_t)q * np + row], am[j], rowfac);
                const double ba = wsr[L.betap + (size_t)a * np + row];
                if (DIAG) { bn[j] = ba; rf[j] = rowfac; ikrow[j] = p.gp.iK + ((size_t)a * p.gp.ldk + row) * p.gp.ldk; }
                else rf[j] = ba * rowfac;
            }
        }
        for (int c0 = 0; c0 < ncol8; c0 += CM) {
            const int cm = (np - c0) < CM ? (np - c0) : CM;
            const int cend = (ncol8 - c0) < cm ? (ncol8 - c0) : cm;
            if (staged) {
                mbar_wait(bar, phase); phase ^= 1; staged = false;
            } else if (!single) {
                __syncthreads();
                if (tid == 0) issue_chunk(c0, false);
                mbar_wait(bar, phase); phase ^= 1;
            }
            if (nlive == 2) tape_sweep<KS, DIAG, 2>(sZ, sBq, sBe, tab, 0, cend, c0, ua, am, rf, bn, ikrow, hl, hz, sCsw, lane);
            else if (nlive == 1) tape_sweep<KS, DIAG, 1>(sZ, sBq, sBe, tab, 0, cend, c0, ua, am, rf, bn, ikrow, hl, hz, sCsw, lane);
        }
        // row-side results of this pass
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            if (oct[j] >= NS) continue;                         // warp-uniform
            double v = 0.0;
            if (oct[j] < NO) {
                const int row = 8 * oct[j] + g;
                constexpr bool ONES = (KS & 1) != 0;
                constexpr int tsum = ONES ? 2 : 0;              // lane of the quad that holds the row sum
                double h;
                if (ONES) h = hz[j][NT - 1][0];                 // HZ[:, DP] (ones column of the second product)
                else {
                    h = hl[j];
                    h += __shfl_xor_sync(0xffffffffu, h, 1);
                    h += __shfl_xor_sync(0xffffffffu, h, 2);
                }
                const double hrv = rf[j] * h;
                if (t == tsum) { tpr[TL.hr + (size_t)q * np + row] = hrv; v = hrv; }
                double* hzrow = tpr + TL.HZ + ((size_t)q * np + row) * ldz;      // (TL.ldh == ldz)
#pragma unroll
                for (int nt = 0; nt < NT; ++nt)
                    if (8 * nt + 2 * t < ldz)                                    // columns beyond the row stride: not stored
                        *reinterpret_cast<double2*>(hzrow + 8 * nt + 2 * t) = make_double2(rf[j] * hz[j][nt][0], rf[j] * hz[j][nt][1]);
                v = warp_sum(v);
            }
            if (lane == 0) p.ws[(size_t)r * L.per_r + L.Tpart + (size_t)q * NS + oct[j]] = v;
        }
    }
    // column sums of this CTA's rows: fixed order over the warps (deterministic); not produced for the diagonal pairs of
    // an exact GP (symmetric H: the finish task takes hr in their place, mm_tape_pair_is_symmetric)
    if (!DIAG) {
        __syncthreads();
        double* hc = tpr + TL.hc + ((size_t)q * cs + sidx) * np;
        for (int c = tid; c < np; c += blockDim.x) {
            double v = 0.0;
#pragma unroll
            for (int w = 0; w < 8; ++w) v += sCs[(size_t)w * np + c];
            hc[c] = v;
        }
    }
}

// LB = the thread count promised to the compiler (the launch uses 256): with 2 CTAs per SM it caps the registers at
// 65536 / (2 LB) -- 304 -> 96 registers (2 CTAs/SM leave 16 k registers per SM for the latency-bound glue kernels of
// the other sub-batches to run BESIDE the tile CTAs), 352 -> 80 registers (3 CTAs/SM fit).  No variant spills.
template <int KS, int LB>
__global__ void __launch_bounds__(LB, 2) mm_tape_tile_kernel(MMParams p) {
    PDL_ENTRY();
    int a, b;
    pair_decode(blockIdx.y, a, b);
    if (a == b && p.gp.mode == 0 && p.gp.iK != nullptr) mm_tape_body<KS, true>(p);
    else mm_tape_body<KS, false>(p);
}

// -------------------------------------------------------------------------------------------------
// The same taped pass on Hopper's native 16x8 MMA shapes: the warp's two row octets are one 16-row tile.
//   exponent  C(16x8) = [B, B] + [U'_o0; U'_o1] . zeta[pi(cols)]   one MMA per K chunk (mma16_k)
//   H.[Z,1]   the exponent's C fragment (c0, c2, c1, c3) of the weighted tile w is the A fragment of m16n8k8 -- (g, t),
//             (g + 8, t), (g, t + 4), (g + 8, t + 4) -- because the exponent's B fragment takes the centres in the order
//             pi; its B fragments are tape_sweep's zb[0][nt], zb[1][nt]: ONE DMMA.16x8x8 per n-tile, no shuffles.
// hz[nt][0..1] = row g of octet 0, hz[nt][2..3] = row g of octet 1 (columns 8 nt + 2t, 8 nt + 2t + 1).  A dead second
// octet (ua = 0, rf = 0) rides along; its sums are dropped.
// -------------------------------------------------------------------------------------------------
template <int KS, bool DIAG>
__device__ __forceinline__ void tape_sweep_m16(const double* __restrict__ sZ, const double* __restrict__ sBq,
                                               const double* __restrict__ sBe, const double* __restrict__ tab,
                                               int cbeg, int cend, int c0,
                                               const double (&af)[2 * KS], const double (&am)[2], const double (&rf)[2],
                                               const double (&bn)[2], const double* const (&ikrow)[2],
                                               double (&hl)[2], double (&hz)[(4 * KS + 7) / 8][4],
                                               double* __restrict__ sCsw, int lane) {
    constexpr int ldz = KS == 1 ? 4 : (KS <= 3 ? 12 : 20);
    constexpr int NT = (4 * KS + 7) / 8;
    constexpr bool ONES = (KS & 1) != 0;                       // DP = 4 KS = 4 (mod 8)
    const int g = lane >> 2, t = lane & 3;
    const int pg = (g >> 1) | ((g & 1) << 2);                  // pi(g)
    const double* ltab = EXP_LANE_TAB(tab, lane);
    for (int cg = cbeg; cg < cend; cg += 8) {
        const double bq0 = sBq[cg + t], bq1 = sBq[cg + 4 + t];
        const double bb0 = sBe[cg + t], bb1 = sBe[cg + 4 + t];
        double bf[KS];
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) bf[ks] = sZ[(size_t)(cg + pg) * ldz + 4 * ks + t];
        double zb[2][NT];
#pragma unroll
        for (int k2 = 0; k2 < 2; ++k2)
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) zb[k2][nt] = sZ[(size_t)(cg + 4 * k2 + t) * ldz + 8 * nt + g];
        if (ONES && g == 4) { zb[0][NT - 1] = 1.0; zb[1][NT - 1] = 1.0; }   // ones column: row sums as HZ[:, DP]
        double e[4] = {bq0, bq1, bq0, bq1};
        mma16_k<KS>(e, af, bf);
        double w[4];                                            // A fragment of H.[Z,1]: w0(o0), w0(o1), w1(o0), w1(o1)
        double cs0 = 0.0, cs1 = 0.0;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const double l0 = exp_shifted(e[2 * j], am[j], ltab), l1 = exp_shifted(e[2 * j + 1], am[j], ltab);
            double w0, w1;
            if (DIAG) {
                const double ik0 = ikrow[j][c0 + cg + t], ik1 = ikrow[j][c0 + cg + 4 + t];   // zero padded: in bounds
                w0 = fma(bn[j], bb0, -ik0) * l0;
                w1 = fma(bn[j], bb1, -ik1) * l1;
            } else {
                w0 = bb0 * l0; w1 = bb1 * l1;
            }
            if (!ONES) hl[j] += w0 + w1;
            if (!DIAG) { cs0 = fma(rf[j], w0, cs0); cs1 = fma(rf[j], w1, cs1); }
            w[j] = w0; w[2 + j] = w1;
        }
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) dmma1688(hz[nt], w, zb[0][nt], zb[1][nt]);
        if (!DIAG) {                                            // column sums: the reduce-scatter butterfly of tape_sweep
            const bool up = (g & 4) != 0;
            double keep = up ? cs1 : cs0;
            const double send = up ? cs0 : cs1;
            keep += __shfl_xor_sync(0xffffffffu, send, 16);
            keep += __shfl_xor_sync(0xffffffffu, keep, 8);
            keep += __shfl_xor_sync(0xffffffffu, keep, 4);
            if ((g & 3) == 0) sCsw[c0 + cg + (up ? 4 : 0) + t] += keep;
        }
    }
}

// CTA = (row split, pair, restart) as mm_tape_body.  A pass whose second block of octets is past the last row (at the
// bench shapes: the last pass of every pair) does not fall back to one octet per warp: warps 0-3 take the octet pairs
// {2w, 2w + 1} of the remaining block over all columns, warps 4-7 have no rows in that pass.  An octet's row-side results
// (hr, HZ, T) are the same whichever pass form it ran in, so they do not depend on the row splits (i.e. the batch size).
// The column sums hc do: they are stored per row split and added up by the reverse sweep (DESIGN.md section 4).
template <int KS, bool DIAG>
__device__ __forceinline__ void mm_tape_body_m16(const MMParams& p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int ldz = KS == 1 ? 4 : (KS <= 3 ? 12 : 20);
    constexpr int NT = (4 * KS + 7) / 8;
    const MMWs& L = p.L;
    const MMTapeL& TL = p.TL;
    const int np = L.np, n = p.gp.n;
    const int CM = np < TILE_CM ? np : TILE_CM;
    double* sZ = reinterpret_cast<double*>(smem_raw);
    double* sBq = sZ + (size_t)CM * ldz;
    double* sBe = sBq + CM;
    double* tab = sBe + CM;
    uint64_t* bar = reinterpret_cast<uint64_t*>(tab + EXP_TAB_DOUBLES);
    double* sCs = reinterpret_cast<double*>(bar + 2);          // [8 warps][np] column-sum partials

    const int r = blockIdx.z, q = blockIdx.y, sidx = blockIdx.x, cs = gridDim.x;
    int a, b;
    pair_decode(q, a, b);
    const double* wsr = p.ws + (size_t)r * L.per_r;
    double* tpr = p.tape + (size_t)r * TL.per_r;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int NO = (n + 7) >> 3, NS = np >> 3;                 // live row octets / partial-sum slots of a pair
    const int ncol8 = (n + 7) & ~7;
    const bool single = ncol8 <= CM;
    double* sCsw = sCs + (size_t)warp * np;

    if (tid == 0) { mbar_init(bar, 1); mbar_fence_init(); }
    for (int c = lane; c < np; c += 32) sCsw[c] = 0.0;
    auto issue_chunk = [&](int c0, bool with_table) {
        const int cm = (np - c0) < CM ? (np - c0) : CM;
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
        mbar_expect_tx(bar, (unsigned)(cm * ldz * 8 + cm * 16 + (with_table ? EXP_TAB_DOUBLES * 8 : 0)));
        tma_bulk_g2s(sZ, wsr + L.zeta + (size_t)c0 * ldz, (unsigned)(cm * ldz * 8), bar);
        tma_bulk_g2s(sBq, wsr + L.Bq + (size_t)q * np + c0, (unsigned)(cm * 8), bar);
        tma_bulk_g2s(sBe, wsr + L.betap + (size_t)b * np + c0, (unsigned)(cm * 8), bar);
        if (with_table) tma_bulk_g2s(tab, g_exp_tab, (unsigned)(EXP_TAB_DOUBLES * 8), bar);
    };
    __syncthreads();                                    // barrier initialised before the first arrive / wait
    if (tid == 0) issue_chunk(0, true);

    const int GW = cs * 8, gw = sidx * 8 + warp;
    const int npass = (NS + 2 * GW - 1) / (2 * GW);     // uniform over the CTA (barriers inside when !single)
    unsigned phase = 0;
    bool staged = true;
    for (int pass = 0; pass < npass; ++pass) {
        // octet blocks of this pass: sidx * 8 + (2 pass) GW + [0, 8) and sidx * 8 + (2 pass + 1) GW + [0, 8)
        const int base0 = sidx * 8 + (2 * pass) * GW;
        const bool odd = base0 < NO && base0 + GW >= NO;       // uniform over the CTA: the second block is past the rows
        int oct[2];
        if (!odd) { oct[0] = gw + (2 * pass) * GW; oct[1] = gw + (2 * pass + 1) * GW; }
        else if (warp < 4) { oct[0] = base0 + 2 * warp; oct[1] = oct[0] + 1; }
        else { oct[0] = oct[1] = NS; }                         // no rows (no loads, no sweep, no outputs)
        double af[2 * KS], am[2], rf[2], bn[2], hl[2], hz[NT][4];
        const double* ikrow[2];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) { hz[nt][0] = hz[nt][1] = hz[nt][2] = hz[nt][3] = 0.0; }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            hl[j] = 0.0; bn[j] = 0.0; rf[j] = 0.0; am[j] = EXP_MAGIC; ikrow[j] = nullptr;
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) af[2 * ks + j] = 0.0;
            if (oct[j] < NO) {
                const int row = 8 * oct[j] + g;
                const double* uf = wsr + L.Ufrag + ((size_t)q * NS + oct[j]) * (KS * 32);
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) af[2 * ks + j] = uf[ks * 32 + lane];
                double rowfac;
                exp_row_split(wsr[L.Arow + (size_t)q * np + row], am[j], rowfac);
                const double ba = wsr[L.betap + (size_t)a * np + row];
                if (DIAG) { bn[j] = ba; rf[j] = rowfac; ikrow[j] = p.gp.iK + ((size_t)a * p.gp.ldk + row) * p.gp.ldk; }
                else rf[j] = ba * rowfac;
            }
        }
        if (DIAG && ikrow[1] == nullptr) ikrow[1] = ikrow[0];  // dead second octet: any readable row (its sums are dropped)
        const bool live = oct[0] < NO;                         // warp-uniform
        for (int c0 = 0; c0 < ncol8; c0 += CM) {
            const int cm = (np - c0) < CM ? (np - c0) : CM;
            const int cend = (ncol8 - c0) < cm ? (ncol8 - c0) : cm;
            if (staged) {
                mbar_wait(bar, phase); phase ^= 1; staged = false;
            } else if (!single) {
                __syncthreads();
                if (tid == 0) issue_chunk(c0, false);
                mbar_wait(bar, phase); phase ^= 1;
            }
            if (live) tape_sweep_m16<KS, DIAG>(sZ, sBq, sBe, tab, 0, cend, c0, af, am, rf, bn, ikrow, hl, hz, sCsw, lane);
        }
        // row-side results of this pass
        {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                if (oct[j] >= NS) continue;                     // warp-uniform
                double v = 0.0;
                if (oct[j] < NO) {
                    const int row = 8 * oct[j] + g;
                    constexpr bool ONES = (KS & 1) != 0;
                    constexpr int tsum = ONES ? 2 : 0;          // lane of the quad that holds the row sum
                    double h;
                    if (ONES) h = hz[NT - 1][2 * j];            // HZ[:, DP] (ones column of the second product)
                    else {
                        h = hl[j];
                        h += __shfl_xor_sync(0xffffffffu, h, 1);
                        h += __shfl_xor_sync(0xffffffffu, h, 2);
                    }
                    const double hrv = rf[j] * h;
                    if (t == tsum) { tpr[TL.hr + (size_t)q * np + row] = hrv; v = hrv; }
                    double* hzrow = tpr + TL.HZ + ((size_t)q * np + row) * ldz;      // (TL.ldh == ldz)
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt)
                        if (8 * nt + 2 * t < ldz)                                // columns beyond the row stride: not stored
                            *reinterpret_cast<double2*>(hzrow + 8 * nt + 2 * t) = make_double2(rf[j] * hz[nt][2 * j], rf[j] * hz[nt][2 * j + 1]);
                    v = warp_sum(v);
                }
                if (lane == 0) p.ws[(size_t)r * L.per_r + L.Tpart + (size_t)q * NS + oct[j]] = v;
            }
        }
    }
    // column sums of this CTA's rows: fixed order over the warps (deterministic); none for the diagonal pairs of an exact GP
    if (!DIAG) {
        __syncthreads();
        double* hc = tpr + TL.hc + ((size_t)q * cs + sidx) * np;
        for (int c = tid; c < np; c += blockDim.x) {
            double v = 0.0;
#pragma unroll
            for (int w = 0; w < 8; ++w) v += sCs[(size_t)w * np + c];
            hc[c] = v;
        }
    }
}

// 2 CTAs/SM (<= 128 registers, as mm_tape_tile_kernel<KS, 256>)
template <int KS>
__global__ void __launch_bounds__(256, 2) mm_tape_tile_m16_kernel(MMParams p) {
    PDL_ENTRY();
    int a, b;
    pair_decode(blockIdx.y, a, b);
    if (a == b && p.gp.mode == 0 && p.gp.iK != nullptr) mm_tape_body_m16<KS, true>(p);
    else mm_tape_body_m16<KS, false>(p);
}

#endif  // __CUDACC__

// taped tile pass in place of mm_tile_kernel (p.tape != nullptr); defined in mm_tape.cu
int mm_tape_tile_launch(const MMParams& p, cudaStream_t st);

// reverse sweep from the tape (need_param = 0: cotangents of the input moments only)
struct MMTapeBwd {
    pilco_gp_model gp; int R;
    const double* m; const double* s; long long m_rs, s_rs;      // forward inputs
    const double* Mfwd;                                          // forward output M [R,E]
    const double* gM; const double* gS; const double* gV;        // cotangents [R,E],[R,E,E],[R,D,E]
    const double* tape; MMTapeL TL;
    double* part;                                                // [R][ntask][MAXD + D*D] task partials
    double* gm; double* gs; long long gm_rs, gs_rs;
    int accumulate;
};
// the reverse sweep of one taped moment match: cotangents gM, gS, gV of its outputs -> gm, gs (overwritten); tape and its
// layout TL as the forward wrote them, part: task partials
static inline MMTapeBwd mm_tape_bwd_params(const pilco_gp_model* gp, int R, const double* m, long long m_rs,
                                           const double* s, long long s_rs, const double* Mfwd, const double* gM,
                                           const double* gS, const double* gV, const double* tape, const MMTapeL& TL,
                                           double* part, double* gm, long long gm_rs, double* gs, long long gs_rs) {
    MMTapeBwd bp{};
    bp.gp = *gp; bp.R = R; bp.m = m; bp.s = s; bp.m_rs = m_rs; bp.s_rs = s_rs;
    bp.Mfwd = Mfwd; bp.gM = gM; bp.gS = gS; bp.gV = gV; bp.tape = tape; bp.TL = TL;
    bp.part = part; bp.gm = gm; bp.gs = gs; bp.gm_rs = gm_rs; bp.gs_rs = gs_rs; bp.accumulate = 0;
    return bp;
}
static inline __host__ __device__ size_t mm_tape_bwd_part_doubles(int D, int E) {
    return (size_t)(E + npairs_of(E)) * (MAXD + (size_t)D * D);
}
#define TB_THREADS 128
#define TB_WARPS 4
#define TAPE_MAX_CS 4
// dynamic shared memory of the finish tasks: per-centre weights u, v [2][np], then the staged tape slice of the pair
// (HZ [np][ldh] and the column-sum splits [cs][np], fetched by ONE round of TMA bulk copies) which the cross-warp
// reduction buffer [3][NACC][32] re-uses once the k-loop is over
static inline __host__ __device__ size_t mm_tape_bfinish_smem_bytes(int np, int D) {
    const int dp = 4 * ksteps_of(D), tx = (dp + 8) / 8;
    const size_t nacc = 2 * (tx * (tx + 1) + tx * tx);
    const size_t stage = (size_t)np * ldz_of(D) + (size_t)TAPE_MAX_CS * np, red = (size_t)(TB_WARPS - 1) * nacc * 32;
    return ((size_t)2 * np + (stage > red ? stage : red)) * sizeof(double);
}
// with_reduce = false: the caller's next kernel sums the task partials itself (mm_tape_reduce_device)
int mm_tape_backward_launch(const MMTapeBwd& bp, cudaStream_t st, bool with_reduce);
// shapes the taped path supports: the tile kernel keeps 8 x np column sums, the finish tasks stage a pair's tape slice
// -- both in shared memory (n <= 1024 centres for D <= 12, <= 704 beyond; larger models use the recomputing sweep)
static inline __host__ __device__ bool mm_tape_supported(int n, int D) {
    return pad64(n) <= TAPE_MAX_NP && mm_tape_bfinish_smem_bytes(pad64(n), D) + 24 * 1024 <= 220 * 1024
           && mm_tape_smem_bytes(pad64(n), ldz_of(D)) <= PILCO_MAX_SMEM_OPTIN;
}

#ifdef __CUDACC__
// sum of the task partials of one restart -> gm [D], gs [D,D] (symmetrised); all threads of the CTA take part.
// Fixed order over the tasks (deterministic); 4 independent partial sums per element hide the load latency.
__device__ __forceinline__ void mm_tape_reduce_device(const double* __restrict__ part, int ntask, int D,
                                                      double* __restrict__ gm, double* __restrict__ gs, int accumulate) {
    const size_t stride = MAXD + (size_t)D * D;
    for (int e = threadIdx.x; e < D + D * D; e += blockDim.x) {
        double v0 = 0.0, v1 = 0.0, v2 = 0.0, v3 = 0.0;
        if (e < D) {
            const double* p0 = part + e;
            int tk = 0;
#pragma unroll 4
            for (; tk + 3 < ntask; tk += 4) {                        // (unrolled: 16 independent loads in flight)
                v0 += p0[(size_t)tk * stride]; v1 += p0[(size_t)(tk + 1) * stride];
                v2 += p0[(size_t)(tk + 2) * stride]; v3 += p0[(size_t)(tk + 3) * stride];
            }
            for (; tk < ntask; ++tk) v0 += p0[(size_t)tk * stride];
            const double v = (v0 + v1) + (v2 + v3);
            gm[e] = accumulate ? gm[e] + v : v;
        } else {
            const int k = e - D, i = k / D, j = k % D;
            const double* p0 = part + MAXD + i * D + j;
            const double* p1 = part + MAXD + j * D + i;
            int tk = 0;
#pragma unroll 8
            for (; tk + 1 < ntask; tk += 2) {                        // (unrolled: 32 independent loads in flight)
                v0 += p0[(size_t)tk * stride]; v1 += p1[(size_t)tk * stride];
                v2 += p0[(size_t)(tk + 1) * stride]; v3 += p1[(size_t)(tk + 1) * stride];
            }
            for (; tk < ntask; ++tk) { v0 += p0[(size_t)tk * stride]; v1 += p1[(size_t)tk * stride]; }
            const double v = 0.5 * ((v0 + v1) + (v2 + v3));
            gs[k] = accumulate ? gs[k] + v : v;
        }
    }
}

// -------------------------------------------------------------------------------------------------
// reverse sweep from the tape: one CTA (4 warps) per task
//   task <  E : mean / V block of output a   (per-centre weights recomputed: n exps, W-form of mgpr.py:103-118)
//   task >= E : covariance block of the unordered pair q = task - E, from hr, hc, HZ on the tape
// Both reduce to weighted moment sums over the centres; with zx_n = [zeta_n, 1] (the 1 at index D) they are the three
// products   zx' diag(u) zx,   zx' diag(v) zx,   zx' HZ   (K = n), evaluated with fp64 DMMA m8n8k4: the k-steps (4
// centres each) are dealt round-robin to the warps, one value zx[row t][col g] per lane serves as A fragment
// (A[m=col][k=row]) AND, scaled by u / v, as B fragment (B[k=row][n=col]).  A1 = block[:D,:D], y1 = block[:D, D],
// sum u = block[D, D]; the symmetric blocks skip their lower tiles.
// -------------------------------------------------------------------------------------------------

template <int DP>
__device__ __forceinline__ void mm_tape_bfinish_task(const MMTapeBwd& bp, int r, int task, double* tb_dyn) {
    // tb_dyn (dynamic shared memory): [2][np] per-centre weights u, v, then the cross-warp reduction buffer
    const pilco_gp_model& gp = bp.gp;
    const MMTapeL& TL = bp.TL;
    const int n = gp.n, D = gp.D, E = gp.E, np = TL.np;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    constexpr int TX = (DP + 8) / 8;                            // 8-wide tiles covering [zeta, 1]: D + 1 <= 8 TX
    constexpr int DX = 8 * TX;
    constexpr int NSYMT = TX * (TX + 1) / 2;                    // upper tiles of a symmetric block
    constexpr int NACC = 2 * (2 * NSYMT + TX * TX);             // accumulator doubles per lane

    __shared__ double sW[MAXD * SLD], sCm[MAXD * SLD], sT[MAXD * SLD], sX[MAXD * SLD];
    __shared__ double sinvd[MAXD], spa[MAXD], spb[MAXD], sgv[MAXD], swgv[MAXD], sm[MAXD];
    __shared__ double sA1[DX * DX], sA2[DX * DX], sA3[DX * DX], sscal[4];
    double* su = tb_dyn;
    double* sv = tb_dyn + np;
    double* sHZ = tb_dyn + 2 * (size_t)np;                     // staged HZ slice of the pair [np][ldh] ...
    double* sHc = sHZ + (size_t)np * TL.ldh;                   // ... and its column-sum splits [cs][np]
    double* sRed = sHZ;                                        // [(TB_WARPS - 1)][NACC][32]: re-uses the staging area after the k-loop
    __shared__ __align__(8) uint64_t tbar;

    const double* X = gp.X + (size_t)r * gp.X_bs;
    const double* ell = gp.ell + (size_t)r * gp.ell_bs;
    const double* sf2 = gp.sf2 + (size_t)r * gp.sf2_bs;
    const double* beta = gp.beta + (size_t)r * gp.beta_bs;
    const double* mr = bp.m + (size_t)r * bp.m_rs;
    const double* sr = bp.s + (size_t)r * bp.s_rs;
    const double* gS = bp.gS + (size_t)r * E * E;
    const double* tpr = bp.tape + (size_t)r * TL.per_r;
    double* part = bp.part + ((size_t)r * (E + TL.P) + task) * (MAXD + (size_t)D * D);
    double* Tm = part;
    double* Ts = part + MAXD;
    if (tid < MAXD) sm[tid] = tid < D ? mr[tid] : 0.0;

    const bool is_out = task < E;
    int a = task, b = task, q = 0;
    const double* HZg = nullptr;
    if (is_out) {
        // ---- output task: W_a = (s + Lambda_a^2)^-1, c_a, per-centre weights u_n = gw_n w_n, v_n = w_n ----
        if (tid < DP) {
            const double l = tid < D ? ell[a * D + tid] : 1.0;
            spa[tid] = l * l;
            double gv = 0.0;
            if (tid < D) {
                if (bp.gV) gv = bp.gV[((size_t)r * D + tid) * E + a];
                else                       // rollout glue folded in: gV = s1' (gS + gS'), s1 = first E rows of the joint covariance
                    for (int i = 0; i < E; ++i) gv = fma(sr[i * D + tid], gS[i * E + a] + gS[a * E + i], gv);
            }
            sgv[tid] = gv;
        }
        __syncthreads();
        for (int e = tid; e < DP * DP; e += blockDim.x) {
            const int i = e / DP, j = e % DP;
            const double sij = (i < D && j < D) ? 0.5 * (sr[i * D + j] + sr[j * D + i]) : 0.0;
            sT[i * SLD + j] = sij + (i == j ? spa[i] : 0.0);
            sW[i * SLD + j] = (i == j) ? 1.0 : 0.0;
        }
        __syncthreads();
        if (warp == 0) {
            chol_warp(sT, sinvd, DP, lane);
            chol_solve_warp(sT, sinvd, sW, DP, DP, lane);
            if (lane == 0) {
                double ld = chol_logdet(sinvd, DP), sl = 0.0;
                for (int d = 0; d < D; ++d) sl += log(spa[d]);
                sscal[0] = exp(log(sf2[a]) + 0.5 * (sl - ld));           // c_a
                double gmt = bp.gM[(size_t)r * E + a];                   // gMtot[a] = gM[a] - sum_b (gS[a,b]+gS[b,a]) M_b
                for (int bb = 0; bb < E; ++bb) gmt -= (gS[a * E + bb] + gS[bb * E + a]) * bp.Mfwd[(size_t)r * E + bb];
                sscal[1] = gmt;
            }
        }
        __syncthreads();
        if (tid < DP) {                       // W gV_a
            double v = 0.0;
            for (int j = 0; j < DP; ++j) v = fma(sW[tid * SLD + j], sgv[j], v);
            swgv[tid] = v;
        }
        __syncthreads();
        const double ca = sscal[0], gmt = sscal[1];
        for (int nn = tid; nn < np; nn += blockDim.x) {
            double u = 0.0, v = 0.0;
            if (nn < n) {
                double z[DP];
#pragma unroll
                for (int d = 0; d < DP; ++d) z[d] = d < D ? X[(size_t)nn * D + d] - sm[d] : 0.0;
                double e = 0.0, tg = 0.0;
#pragma unroll 1
                for (int i = 0; i < D; ++i) {                            // (rolled: keeps W out of the registers)
                    double ti = 0.0;
#pragma unroll
                    for (int j = 0; j < DP; ++j) ti = fma(sW[i * SLD + j], z[j], ti);
                    const double zi = X[(size_t)nn * D + i] - sm[i];
                    e = fma(zi, ti, e);
                    tg = fma(zi, swgv[i], tg);                           // t_n . gV_a = zeta_n . (W gV_a)
                }
                v = beta[(size_t)a * n + nn] * exp(-0.5 * e) * ca;       // w_n
                u = (gmt + tg) * v;                                      // gw_n w_n
            }
            su[nn] = u; sv[nn] = v;
        }
    } else {
        // ---- pair task: the pair's slice of the tape -- hr, the column-sum splits and HZ -- comes in by ONE round of TMA
        // bulk copies (the tape was written a whole rollout ago: DRAM-cold; a single bulk round trip instead of a
        // dependent global load per k-step); Q, C are fetched meanwhile
        q = task - E;
        pair_decode(q, a, b);
        if (tid == 0) { mbar_init(&tbar, 1); mbar_fence_init(); }
        __syncthreads();
        // diagonal pair of an exact GP: H is symmetric, the tile kernel left no column sums (hc = hr)
        const bool symh = a == b && gp.mode == 0 && gp.iK != nullptr;
        if (tid == 0) {
            const unsigned bhz = (unsigned)((size_t)n * TL.ldh * 8), bhr = (unsigned)(np * 8), bhc = symh ? 0u : (unsigned)((size_t)TL.cs * np * 8);
            mbar_expect_tx(&tbar, bhz + bhr + bhc);
            tma_bulk_g2s(sHZ, tpr + TL.HZ + (size_t)q * np * TL.ldh, bhz, &tbar);
            tma_bulk_g2s(su, tpr + TL.hr + (size_t)q * np, bhr, &tbar);
            if (!symh) tma_bulk_g2s(sHc, tpr + TL.hc + (size_t)q * TL.cs * np, bhc, &tbar);
        }
        if (tid < DP) {
            const double la = tid < D ? ell[a * D + tid] : 1.0, lb = tid < D ? ell[b * D + tid] : 1.0;
            spa[tid] = tid < D ? 1.0 / (la * la) : 0.0;
            spb[tid] = tid < D ? 1.0 / (lb * lb) : 0.0;
        }
        const double* Qg = tpr + TL.Q + (size_t)q * D * D;
        const double* Cg = tpr + TL.C + (size_t)q * D * D;
        for (int e = tid; e < DP * DP; e += blockDim.x) {
            const int i = e / DP, j = e % DP;
            const bool in = i < D && j < D;
            sW[i * SLD + j] = in ? Qg[i * D + j] : 0.0;
            sCm[i * SLD + j] = in ? Cg[i * D + j] : 0.0;
        }
        mbar_wait(&tbar, 0);
        // v = sum of the row splits of the column sums; rows at or beyond n carry no weight (the tile kernel never wrote them)
        for (int nn = tid; nn < np; nn += blockDim.x) {
            double v = 0.0;
            if (nn < n) {
                if (symh) v = su[nn];
                else for (int k = 0; k < TL.cs; ++k) v += sHc[(size_t)k * np + nn];
            } else su[nn] = 0.0;
            sv[nn] = v;
        }
        HZg = sHZ;                                               // (shared memory from here on)
    }
    __syncthreads();

    // ---- weighted moment sums by DMMA ----
    double cu[NSYMT][2], cv[NSYMT][2], ch[TX * TX][2];
#pragma unroll
    for (int i = 0; i < NSYMT; ++i) { cu[i][0] = cu[i][1] = cv[i][0] = cv[i][1] = 0.0; }
#pragma unroll
    for (int i = 0; i < TX * TX; ++i) { ch[i][0] = ch[i][1] = 0.0; }
    // TBU k-steps per trip: their centres X (global memory, L2) are fetched first -- independent loads, one round trip
    // per trip -- then the DMMAs run with the weights and the HZ slice read from shared memory
    constexpr int TBU = (TX <= 2) ? 8 : 4;
    const int nks = (n + 3) >> 2;
    for (int ks0 = warp; ks0 < nks; ks0 += TB_WARPS * TBU) {
        double zx[TBU][TX];
#pragma unroll
        for (int k = 0; k < TBU; ++k) {
            const int row = 4 * (ks0 + k * TB_WARPS) + t;
#pragma unroll
            for (int tl = 0; tl < TX; ++tl) {
                const int c = g + 8 * tl;
                zx[k][tl] = (row < n && c < D) ? X[(size_t)row * D + c] : 0.0;
            }
        }
#pragma unroll
        for (int k = 0; k < TBU; ++k) {
            const int row = 4 * (ks0 + k * TB_WARPS) + t;
            if (4 * (ks0 + k * TB_WARPS) >= n) break;             // warp-uniform: no k-step left
            const bool live = row < n;
            const double uk = live ? su[row] : 0.0, vk = live ? sv[row] : 0.0;
            double bu[TX], bv[TX], bh[TX];
#pragma unroll
            for (int tl = 0; tl < TX; ++tl) {
                const int c = g + 8 * tl;
                double z = 0.0, h = 0.0;
                if (live) {
                    if (c < D) { z = zx[k][tl] - sm[c]; if (HZg) h = HZg[(size_t)row * TL.ldh + c]; }
                    else if (c == D) z = 1.0;
                }
                zx[k][tl] = z; bu[tl] = uk * z; bv[tl] = vk * z; bh[tl] = h;
            }
            int si = 0;
#pragma unroll
            for (int mt = 0; mt < TX; ++mt)
#pragma unroll
                for (int nt = 0; nt < TX; ++nt) {
                    if (nt >= mt) {
                        dmma884(cu[si][0], cu[si][1], zx[k][mt], bu[nt]);
                        dmma884(cv[si][0], cv[si][1], zx[k][mt], bv[nt]);
                        ++si;
                    }
                    if (!is_out) dmma884(ch[mt * TX + nt][0], ch[mt * TX + nt][1], zx[k][mt], bh[nt]);
                }
        }
    }
    // cross-warp reduction (fixed order), then warp 0 scatters the C fragments into square matrices
    __syncthreads();                                           // every warp is done reading the staged slice (sRed aliases it)
    if (warp > 0) {
        double* dst = sRed + ((size_t)(warp - 1) * NACC) * 32 + lane;
        int k = 0;
#pragma unroll
        for (int i = 0; i < NSYMT; ++i) { dst[32 * k++] = cu[i][0]; dst[32 * k++] = cu[i][1]; dst[32 * k++] = cv[i][0]; dst[32 * k++] = cv[i][1]; }
#pragma unroll
        for (int i = 0; i < TX * TX; ++i) { dst[32 * k++] = ch[i][0]; dst[32 * k++] = ch[i][1]; }
    }
    __syncthreads();
    if (warp == 0) {
        for (int w = 0; w < TB_WARPS - 1; ++w) {
            const double* src = sRed + ((size_t)w * NACC) * 32 + lane;
            int k = 0;
#pragma unroll
            for (int i = 0; i < NSYMT; ++i) { cu[i][0] += src[32 * k++]; cu[i][1] += src[32 * k++]; cv[i][0] += src[32 * k++]; cv[i][1] += src[32 * k++]; }
#pragma unroll
            for (int i = 0; i < TX * TX; ++i) { ch[i][0] += src[32 * k++]; ch[i][1] += src[32 * k++]; }
        }
        int si = 0;
#pragma unroll
        for (int mt = 0; mt < TX; ++mt)
#pragma unroll
            for (int nt = 0; nt < TX; ++nt) {
                const int i = 8 * mt + g, j = 8 * nt + 2 * t;
                if (nt >= mt) {
                    sA1[i * DX + j] = cu[si][0]; sA1[i * DX + j + 1] = cu[si][1];
                    sA2[i * DX + j] = cv[si][0]; sA2[i * DX + j + 1] = cv[si][1];
                    if (nt > mt) {
                        sA1[j * DX + i] = cu[si][0]; sA1[(j + 1) * DX + i] = cu[si][1];
                        sA2[j * DX + i] = cv[si][0]; sA2[(j + 1) * DX + i] = cv[si][1];
                    }
                    ++si;
                }
                sA3[i * DX + j] = ch[mt * TX + nt][0]; sA3[i * DX + j + 1] = ch[mt * TX + nt][1];
            }
    }
    __syncthreads();
    // A1 = sA1[:D,:D] etc.; y1[i] = sA1[i][D], y2[i] = sA2[i][D]; sum u = sA1[D][D], sum v = sA2[D][D]
    const double sum_u = sA1[D * DX + D], sum_v = sA2[D * DX + D];

    if (is_out) {
        // gW = -0.5 A1 + sym(gV y2');  gA = -W gW W - 0.5 glogc W;  sum gzeta = -W y1 + (sum w) W gV
        const double glogc = sum_u;
        for (int e = tid; e < DP * DP; e += blockDim.x) {
            const int i = e / DP, j = e % DP;
            sT[i * SLD + j] = (i < D && j < D) ? -0.5 * sA1[i * DX + j] + 0.5 * (sgv[i] * sA2[j * DX + D] + sgv[j] * sA2[i * DX + D]) : 0.0;
        }
        __syncthreads();
        for (int e = tid; e < DP * DP; e += blockDim.x) {           // sCm = W gW
            const int i = e / DP, j = e % DP;
            double v = 0.0;
            for (int k = 0; k < DP; ++k) v = fma(sW[i * SLD + k], sT[k * SLD + j], v);
            sCm[i * SLD + j] = v;
        }
        __syncthreads();
        for (int e = tid; e < D * D; e += blockDim.x) {
            const int i = e / D, j = e % D;
            double v = 0.0;
            for (int k = 0; k < DP; ++k) v = fma(sCm[i * SLD + k], sW[k * SLD + j], v);
            Ts[e] = -v - 0.5 * glogc * sW[i * SLD + j];
        }
        if (tid < D) {
            double v = 0.0;
            for (int j = 0; j < D; ++j) v = fma(sW[tid * SLD + j], sA1[j * DX + D], v);
            Tm[tid] = v - sum_v * swgv[tid];                        // -(sum_n gzeta_n)
        }
        return;
    }

    // pair task
    const double gw = (a == b) ? gS[a * E + a] : gS[a * E + b] + gS[b * E + a];
    const double glogR = -0.5 * gw * sum_u;
    for (int e = tid; e < DP * DP; e += blockDim.x) {               // sT = gQ / (delta_i delta_j)
        const int i = e / DP, j = e % DP;
        double v = 0.0;
        if (i < D && j < D) {
            const double gq = gw * (spa[i] * spa[j] * sA1[i * DX + j] + spb[i] * spb[j] * sA2[i * DX + j]
                                    + spa[i] * spb[j] * sA3[i * DX + j] + spa[j] * spb[i] * sA3[j * DX + i]);
            v = gq / ((spa[i] + spb[i]) * (spa[j] + spb[j]));
        }
        sT[i * SLD + j] = v;
    }
    __syncthreads();
    for (int e = tid; e < DP * DP; e += blockDim.x) {               // sX = C (gQ/dd)
        const int i = e / DP, j = e % DP;
        double v = 0.0;
        for (int k = 0; k < D; ++k) v = fma(sCm[i * SLD + k], sT[k * SLD + j], v);
        sX[i * SLD + j] = v;
    }
    __syncthreads();
    for (int e = tid; e < D * D; e += blockDim.x) {                 // gs_pair = 0.5 C (gQ/dd) C + glogR C
        const int i = e / D, j = e % D;
        double v = 0.0;
        for (int k = 0; k < D; ++k) v = fma(sX[i * SLD + k], sCm[k * SLD + j], v);
        Ts[e] = 0.5 * v + glogR * sCm[i * SLD + j];
    }
    if (tid < D) {                                                  // -(sum gzeta) = g (u - 2 delta o Q u),  u = p_a y1 + p_b y2
        double qu = 0.0;
        for (int j = 0; j < D; ++j) qu = fma(sW[tid * SLD + j], spa[j] * sA1[j * DX + D] + spb[j] * sA2[j * DX + D], qu);
        const double u = spa[tid] * sA1[tid * DX + D] + spb[tid] * sA2[tid * DX + D];
        Tm[tid] = gw * (u - 2.0 * (spa[tid] + spb[tid]) * qu);
    }
}

#endif
