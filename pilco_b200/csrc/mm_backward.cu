// mm_backward.cu -- hand-derived VJP of the SE-ARD moment match (the reference differentiates
// pilco/models/mgpr.py:91-149 with TensorFlow autodiff; see oracle/staged.py:mm_backward_staged for the
// numpy statement of exactly this algorithm and DESIGN.md "Backward").
//
//   bsetup  grid (E*E, R)     : mm_setup_kernel<DP,true>: ordered pairs, also stores Q_ab, C_ab, logdetR_ab
//   btile   grid (NB, E*E, R) : recompute L'[n,m] tile-wise; per row n:  hL = sum_m beta_b[m] L',
//                               HVL = sum_m beta_b[m] L' zeta_m  (+ hK, HVK with iK_a[n,m] on diagonal pairs)
//   bfinish grid (E + E*E, R) : per task partial gradients (mean/V block per output, covariance block per pair)
//   breduce grid (R)          : sums the task partials -> gm, gs (+ gX, gbeta, gell for trainable policies)
#include "mm_backward.cuh"

// -------------------------------------------------------------------------------------------------
// backward tile kernel
// -------------------------------------------------------------------------------------------------
static inline __host__ __device__ size_t mm_btile_smem_bytes(int np, int ldz) {
    const int cm = np < TILE_CM ? np : TILE_CM;
    return (size_t)cm * ldz * 8 + (size_t)cm * 16 + EXP_TAB_DOUBLES * 8 + 16;
}

// DIAG = true : grid (NB, E, R), the pairs (a,a) of a GP with trace term (iK-weighted sums as well);
// DIAG = false: grid (NB, E*E, R), every other ordered pair (CTAs of (a,a) pairs that DIAG handles exit at once).
template <int KS, bool DIAG>
__global__ void __launch_bounds__(256, DIAG ? 2 : 4) mm_btile_kernel(MMBwdParams bp) {
    PDL_ENTRY();
    constexpr int DP = 4 * KS;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const MMParams& p = bp.f;
    const MMWs& L = bp.B.F;
    const int np = L.np, ldz = L.ldz, E = p.gp.E;
    const int CM = np < TILE_CM ? np : TILE_CM;
    double* sZ = reinterpret_cast<double*>(smem_raw);
    double* sBq = sZ + (size_t)CM * ldz;
    double* sBe = sBq + CM;
    double* tab = sBe + CM;
    uint64_t* bar = reinterpret_cast<uint64_t*>(tab + EXP_TAB_DOUBLES);

    const int r = blockIdx.z, rb = blockIdx.x;
    const bool has_trace = (p.gp.mode == 0) && (p.gp.iK != nullptr);
    const int q = DIAG ? blockIdx.y * E + blockIdx.y : blockIdx.y;
    const int a = q / E, b = q % E;
    if (!DIAG && a == b && has_trace) return;           // handled by the DIAG instantiation
    double* wsr = p.ws + (size_t)r * bp.B.per_r;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const double* ltab = EXP_LANE_TAB(tab, lane);
    const int row0 = rb * 64 + warp * 8;
    const int row = row0 + g;
    const bool active = row0 < p.gp.n;
    const int ncol8 = (p.gp.n + 7) & ~7;

    TILE_STAMP(0);                                          // (diagnostics build only, see mm_kernels.cuh)
    if (tid == 0) { mbar_init(bar, 1); mbar_fence_init(); }
    __syncthreads();
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
    double ua[KS], Apv;
    tile_row_operands<KS>(wsr + L.Qab + (size_t)q * PAIR_BLK, wsr + L.zeta, ldz, row, row < p.gp.n, lane, ua, Apv);
    const double* ikrow = DIAG ? p.gp.iK + ((size_t)a * p.gp.ldk + row) * p.gp.ldk : nullptr;
    // as in the forward tile kernel: the integer part of A' rides in the exp's rounding constant, the fractional
    // part (rowfac) scales this row's sums once at the end
    double am, rowfac;
    exp_row_split(Apv, am, rowfac);
    TILE_STAMP(1);

    // accumulators: row sums hL (hK) per lane (quad-reduced at the end) and HV in DMMA C-fragment layout:
    // hv[nt][c] = HV[row g][8 nt + 2t + c], complete sums over the columns (the DMMA reduces over k = column)
    constexpr int NT = (DP + 7) / 8;
    double hl = 0.0, hk = 0.0;
    double hvL[NT][2], hvK[DIAG ? NT : 1][2];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) { hvL[nt][0] = hvL[nt][1] = 0.0; if (DIAG) { hvK[nt][0] = hvK[nt][1] = 0.0; } }
    const int qb = lane & ~3;                              // first lane of this quad
    unsigned phase = 0;
    for (int c0 = 0; c0 < ncol8; c0 += CM) {
        const int cm = (np - c0) < CM ? (np - c0) : CM;
        const int cend = (ncol8 - c0) < cm ? (ncol8 - c0) : cm;
        if (c0 != 0) {
            __syncthreads();
            if (tid == 0) issue_chunk(c0, false);
        }
        mbar_wait(bar, phase);
        phase ^= 1;
        if (c0 == 0) TILE_STAMP(2);
        if (active) {
            for (int col = 0; col < cend; col += 8) {
                const double2 bq = *reinterpret_cast<const double2*>(sBq + col + 2 * t);
                double e0 = bq.x, e1 = bq.y;
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) {
                    const double bf = sZ[(size_t)(col + g) * ldz + 4 * ks + t];
                    dmma884(e0, e1, ua[ks], bf);
                }
                const double l0 = exp_shifted(e0, am, ltab), l1 = exp_shifted(e1, am, ltab);
                const double2 bb = *reinterpret_cast<const double2*>(sBe + col + 2 * t);
                const double w0 = bb.x * l0, w1 = bb.y * l1;        // W[g][2t], W[g][2t+1]  (C-fragment layout)
                hl += w0 + w1;
                double v0 = 0.0, v1 = 0.0;
                if (DIAG) {
                    const double2 ik = *reinterpret_cast<const double2*>(ikrow + c0 + col + 2 * t);
                    v0 = ik.x * l0; v1 = ik.y * l1;
                    hk += v0 + v1;
                }
                // HV[8 x DP] += W[8 x 8] . zeta[col : col+8, 0:DP]  as 2 k-steps x NT n-tiles of DMMA
#pragma unroll
                for (int k2 = 0; k2 < 2; ++k2) {
                    // A fragment: W[g][4 k2 + t], held by quad lane 2 k2 + (t >> 1) as element t & 1
                    const int src = qb | (2 * k2 + (t >> 1));
                    const double x0 = __shfl_sync(0xffffffffu, w0, src), x1 = __shfl_sync(0xffffffffu, w1, src);
                    const double aw = (t & 1) ? x1 : x0;
                    double ak = 0.0;
                    if (DIAG) {
                        const double y0 = __shfl_sync(0xffffffffu, v0, src), y1 = __shfl_sync(0xffffffffu, v1, src);
                        ak = (t & 1) ? y1 : y0;
                    }
                    const double* zrow = sZ + (size_t)(col + 4 * k2 + t) * ldz;
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt) {
                        const double bz = (8 * nt + g < DP) ? zrow[8 * nt + g] : 0.0;     // B[k = col][n = d]
                        dmma884(hvL[nt][0], hvL[nt][1], aw, bz);
                        if (DIAG) dmma884(hvK[nt][0], hvK[nt][1], ak, bz);
                    }
                }
            }
        }
    }
    TILE_STAMP(3);
    // outputs per row: [0]=hL, [1..DP]=HVL, [DP+1]=hK, [DP+2..2DP+1]=HVK  (hK/HVK only for DIAG pairs)
    double* out = wsr + bp.B.rowout + ((size_t)q * np + row) * bp.B.ldr;
    hl += __shfl_xor_sync(0xffffffffu, hl, 1);
    hl += __shfl_xor_sync(0xffffffffu, hl, 2);
    if (t == 0) out[0] = active ? hl * rowfac : 0.0;
    if (DIAG) {
        hk += __shfl_xor_sync(0xffffffffu, hk, 1);
        hk += __shfl_xor_sync(0xffffffffu, hk, 2);
        if (t == 0) out[DP + 1] = active ? hk * rowfac : 0.0;
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const int d0 = 8 * nt + 2 * t;
        if (d0 < DP) {
            out[1 + d0] = active ? hvL[nt][0] * rowfac : 0.0;
            out[2 + d0] = active ? hvL[nt][1] * rowfac : 0.0;
            if (DIAG) { out[DP + 2 + d0] = active ? hvK[nt][0] * rowfac : 0.0; out[DP + 3 + d0] = active ? hvK[nt][1] * rowfac : 0.0; }
        }
    }
    TILE_STAMP(4);
}

// -------------------------------------------------------------------------------------------------
// backward finish: one CTA (128 threads) per task
// -------------------------------------------------------------------------------------------------
#define BF_CHUNK 128

template <int DP>
__device__ __forceinline__ void mm_bfinish_task(const MMBwdParams& bp, int r, int task) {
    const MMParams& p = bp.f;
    const pilco_gp_model& gp = p.gp;
    const MMBws& B = bp.B;
    const MMWs& L = B.F;
    const int n = gp.n, D = gp.D, E = gp.E, np = L.np, ldz = L.ldz;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    __shared__ double sW[MAXD * SLD];         // W_a (output task) or Q_ab (pair task)
    __shared__ double sCm[MAXD * SLD];        // C_ab (pair) / scratch
    __shared__ double sT[MAXD * SLD];         // scratch
    __shared__ double sinvd[MAXD];
    __shared__ double spa[MAXD], spb[MAXD], sgv[MAXD], swgv[MAXD];
    __shared__ double sred[(2 * MAXD + 2) * 4], sout[2 * MAXD + 2];
    __shared__ double sOm[MAXD * MAXD];
    __shared__ double sRowA[BF_CHUNK][DP + 1];   // za_n (pair) / (gw w) zeta_n (output)
    __shared__ double sRowB[BF_CHUNK][DP + 1];   // w_n  (pair) / zeta_n (output)
    __shared__ double sscal[4];

    const double* ell = gp.ell + (size_t)r * gp.ell_bs;
    const double* sf2 = gp.sf2 + (size_t)r * gp.sf2_bs;
    const double* beta = gp.beta + (size_t)r * gp.beta_bs;
    double* wsr = p.ws + (size_t)r * B.per_r;
    const double* zeta = wsr + L.zeta;
    const double* gS = bp.gS + (size_t)r * E * E;
    double* Tm = wsr + B.Tm + (size_t)task * MAXD;
    double* Ts = wsr + B.Ts + (size_t)task * D * D;
    double* Tpa = wsr + B.Tpa + (size_t)task * MAXD;
    double* Tpb = wsr + B.Tpb + (size_t)task * MAXD;
    double* Tz = wsr + B.Tz + (size_t)task * np * MAXD;
    double* Tb = wsr + B.Tb + (size_t)task * np;
    for (int e = tid; e < DP * DP; e += blockDim.x) sOm[e] = 0.0;

    if (task < E) {
        // ================= mean / V block of output a =================
        const int a = task;
        const double* sr = p.s + (size_t)r * p.s_rs;
        if (tid < DP) {
            const double l = tid < D ? ell[a * D + tid] : 1.0;
            spa[tid] = l * l;
            sgv[tid] = tid < D ? bp.gV[((size_t)r * D + tid) * E + a] : 0.0;
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
                // gMtot[a] = gM[a] - sum_b (gS[a,b] + gS[b,a]) M_b
                double gmt = bp.gM[(size_t)r * E + a];
                for (int bb = 0; bb < E; ++bb) gmt -= (gS[a * E + bb] + gS[bb * E + a]) * p.M[(size_t)r * E + bb];
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
        double acc[2 * DP + 1];               // [0..DP) sum gzeta, [DP..2DP) y, [2DP] glogc
#pragma unroll
        for (int i = 0; i <= 2 * DP; ++i) acc[i] = 0.0;
        for (int c0 = 0; c0 < np; c0 += BF_CHUNK) {
            const int nn = c0 + tid;
            const int krows = (n - c0) < BF_CHUNK ? (n - c0 > 0 ? n - c0 : 0) : BF_CHUNK;   // staged rows beyond n are zero
            double z[DP], gww = 0.0;
#pragma unroll
            for (int d = 0; d < DP; ++d) z[d] = 0.0;
            if (nn < n) {
                double tt[DP], e = 0.0, tg = 0.0;
#pragma unroll
                for (int d = 0; d < DP; ++d) z[d] = d < ldz ? zeta[(size_t)nn * ldz + d] : 0.0;
#pragma unroll
                for (int i = 0; i < DP; ++i) {
                    double v = 0.0;
#pragma unroll
                    for (int j = 0; j < DP; ++j) v = fma(sW[i * SLD + j], z[j], v);
                    tt[i] = v; e = fma(z[i], v, e); tg = fma(v, sgv[i], tg);
                }
                const double qv = exp(-0.5 * e);
                const double w = beta[(size_t)a * n + nn] * qv * ca;
                const double gw = gmt + tg;
                gww = gw * w;
                acc[2 * DP] += gww;
#pragma unroll
                for (int d = 0; d < DP; ++d) {
                    const double gz = -gww * tt[d] + w * swgv[d];
                    acc[d] += gz;
                    acc[DP + d] = fma(w, z[d], acc[DP + d]);
                    if (bp.need_param) Tz[(size_t)nn * MAXD + d] = gz;
                }
                if (bp.need_param) Tb[nn] = gw * qv * ca;
            } else if (bp.need_param && nn < np) {
                for (int d = 0; d < DP; ++d) Tz[(size_t)nn * MAXD + d] = 0.0;
                Tb[nn] = 0.0;
            }
#pragma unroll
            for (int d = 0; d < DP; ++d) { sRowA[tid][d] = gww * z[d]; sRowB[tid][d] = z[d]; }
            __syncthreads();
            for (int e = tid; e < DP * DP; e += blockDim.x) {       // sum_n (gw w zeta)[i] zeta[j]
                const int i = e / DP, j = e % DP;
                double v = sOm[e];
                for (int k = 0; k < krows; ++k) v = fma(sRowA[k][i], sRowB[k][j], v);
                sOm[e] = v;
            }
            __syncthreads();
        }
        block_sum<2 * MAXD + 2>(acc, 2 * DP + 1, sred, sout);
        const double glogc = sout[2 * DP];
        // gW = -0.5 sOm + sym(gV y^T);  gA = -W gW W - 0.5 glogc W
        for (int e = tid; e < DP * DP; e += blockDim.x) {
            const int i = e / DP, j = e % DP;
            sT[i * SLD + j] = -0.5 * sOm[e] + 0.5 * (sgv[i] * sout[DP + j] + sgv[j] * sout[DP + i]);
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
            const double ga = -v - 0.5 * glogc * sW[i * SLD + j];
            Ts[e] = ga;
            if (i == j) Tpa[i] = ga + 0.5 * glogc / spa[i];         // g(ell_a^2)
        }
        if (tid < DP) { Tm[tid] = -sout[tid]; Tpb[tid] = 0.0; }
        return;
    }

    // ================= covariance block of the ordered pair (a,b), row side =================
    const int q = task - E;
    const int a = q / E, b = q % E;
    const double gt = gS[a * E + b] + gS[b * E + a];
    const double* Qg = wsr + B.oQ + (size_t)q * D * D;
    const double* Cg = wsr + B.oC + (size_t)q * D * D;
    if (tid < DP) {
        const double la = tid < D ? ell[a * D + tid] : 1.0, lb = tid < D ? ell[b * D + tid] : 1.0;
        spa[tid] = tid < D ? 1.0 / (la * la) : 0.0;
        spb[tid] = tid < D ? 1.0 / (lb * lb) : 0.0;
    }
    for (int e = tid; e < DP * DP; e += blockDim.x) {
        const int i = e / DP, j = e % DP;
        const bool in = i < D && j < D;
        sW[i * SLD + j] = in ? Qg[i * D + j] : 0.0;
        sCm[i * SLD + j] = in ? Cg[i * D + j] : 0.0;
    }
    __syncthreads();
    const bool diag = (a == b) && (gp.mode == 0) && (gp.iK != nullptr);
    double acc[2 * DP + 1];                   // [0..DP) sum gzeta_n ; [DP..2DP) row part of g p_a ; [2DP] T
#pragma unroll
    for (int i = 0; i <= 2 * DP; ++i) acc[i] = 0.0;
    for (int c0 = 0; c0 < np; c0 += BF_CHUNK) {
        const int nn = c0 + tid;
        const int krows = (n - c0) < BF_CHUNK ? (n - c0 > 0 ? n - c0 : 0) : BF_CHUNK;       // staged rows beyond n are zero
        double za[DP], wv[DP];
#pragma unroll
        for (int d = 0; d < DP; ++d) { za[d] = 0.0; wv[d] = 0.0; }
        if (nn < n) {
            const double* ro = wsr + B.rowout + ((size_t)q * np + nn) * B.ldr;
            const double ba = beta[(size_t)a * n + nn];
            const double hL = ro[0];
            double hr = ba * hL;
            if (diag) hr -= ro[DP + 1];
            double z[DP];
#pragma unroll
            for (int d = 0; d < DP; ++d) {
                z[d] = d < ldz ? zeta[(size_t)nn * ldz + d] : 0.0;
                double hv = ba * ro[1 + d];
                if (diag) hv -= ro[DP + 2 + d];
                za[d] = spa[d] * z[d];
                wv[d] = hr * za[d] + spb[d] * hv;               // hr za_n + p_b o HV_n
            }
            acc[2 * DP] += hr;
#pragma unroll
            for (int i = 0; i < DP; ++i) {
                double v = 0.0;
#pragma unroll
                for (int j = 0; j < DP; ++j) v = fma(sW[i * SLD + j], wv[j], v);
                const double gza = 2.0 * v;
                const double gz = gt * (spa[i] * gza - hr * za[i]);
                acc[i] += gz;
                acc[DP + i] += gza * z[i] - 0.5 * hr * z[i] * z[i];
                if (bp.need_param) Tz[(size_t)nn * MAXD + i] = gz;
            }
            if (bp.need_param) Tb[nn] = gt * hL;
        } else if (bp.need_param && nn < np) {
            for (int d = 0; d < DP; ++d) Tz[(size_t)nn * MAXD + d] = 0.0;
            Tb[nn] = 0.0;
        }
#pragma unroll
        for (int d = 0; d < DP; ++d) { sRowA[tid][d] = za[d]; sRowB[tid][d] = wv[d]; }
        __syncthreads();
        for (int e = tid; e < DP * DP; e += blockDim.x) {           // Omega^r += sum_n za_n[i] w_n[j]
            const int i = e / DP, j = e % DP;
            double v = sOm[e];
            for (int k = 0; k < krows; ++k) v = fma(sRowA[k][i], sRowB[k][j], v);
            sOm[e] = v;
        }
        __syncthreads();
    }
    block_sum<2 * MAXD + 2>(acc, 2 * DP + 1, sred, sout);
    const double T = sout[2 * DP];
    const double glogR = -0.25 * gt * T;
    // gQ = gt sym(Om) -> sT ;  G2 = gQ / (delta_i delta_j) -> reuse sOm as plain storage after sync
    for (int e = tid; e < DP * DP; e += blockDim.x) {
        const int i = e / DP, j = e % DP;
        sT[i * SLD + j] = 0.5 * gt * (sOm[i * DP + j] + sOm[j * DP + i]);
    }
    __syncthreads();
    // gs_pair = 0.5 C (gQ/dd) C + glogR C
    __shared__ double sX[MAXD * SLD];
    for (int e = tid; e < DP * DP; e += blockDim.x) {               // sX = C (gQ/dd)
        const int i = e / DP, j = e % DP;
        double v = 0.0;
        for (int k = 0; k < D; ++k) {
            const double dk = spa[k] + spb[k], dj = (j < D) ? spa[j] + spb[j] : 1.0;
            v = fma(sCm[i * SLD + k], sT[k * SLD + j] / (dk * dj), v);
        }
        sX[i * SLD + j] = (j < D) ? v : 0.0;
    }
    __syncthreads();
    for (int e = tid; e < D * D; e += blockDim.x) {
        const int i = e / D, j = e % D;
        double v = 0.0;
        for (int k = 0; k < D; ++k) v = fma(sX[i * SLD + k], sCm[k * SLD + j], v);
        Ts[e] = 0.5 * v + glogR * sCm[i * SLD + j];
    }
    // gdelta = -2 diag(Q gQ Q) + 2 glogR diag(Q)
    if (tid < DP) {
        double gd = 0.0;
        if (tid < D) {
            for (int k = 0; k < D; ++k) {
                double v = 0.0;
                for (int l = 0; l < D; ++l) v = fma(sT[k * SLD + l], sW[l * SLD + tid], v);    // (gQ Q)[k][i]
                gd = fma(sW[tid * SLD + k], v, gd);
            }
            gd = -2.0 * gd + 2.0 * glogR * sW[tid * SLD + tid];
        }
        Tm[tid] = -sout[tid];
        Tpa[tid] = gt * sout[DP + tid] + gd;        // contribution to g p_a
        Tpb[tid] = gd;                              // contribution to g p_b
    }
}

// -------------------------------------------------------------------------------------------------
// reduce: sum task partials
// -------------------------------------------------------------------------------------------------
// sum of the task partials of restart r (all threads of one CTA)
__device__ __forceinline__ void mm_breduce_body(const MMBwdParams& bp, int r) {
    const MMParams& p = bp.f;
    const pilco_gp_model& gp = p.gp;
    const MMBws& B = bp.B;
    const int n = gp.n, D = gp.D, E = gp.E, np = B.F.np;
    const int tid = threadIdx.x, nt = blockDim.x;
    const double* wsr = p.ws + (size_t)r * B.per_r;
    const double* ell = gp.ell + (size_t)r * gp.ell_bs;
    double* gm = bp.gm + (size_t)r * bp.gm_rs;
    double* gs = bp.gs + (size_t)r * bp.gs_rs;
    for (int d = tid; d < D; d += nt) {
        double v = 0.0;
        for (int tk = 0; tk < B.ntask; ++tk) v += wsr[B.Tm + (size_t)tk * MAXD + d];
        gm[d] = bp.accumulate ? gm[d] + v : v;
    }
    for (int e = tid; e < D * D; e += nt) {
        const int i = e / D, j = e % D;
        double v = 0.0;
        for (int tk = 0; tk < B.ntask; ++tk)
            v += 0.5 * (wsr[B.Ts + (size_t)tk * D * D + i * D + j] + wsr[B.Ts + (size_t)tk * D * D + j * D + i]);
        gs[e] = bp.accumulate ? gs[e] + v : v;
    }
    if (!bp.need_param) return;
    double* gX = bp.gX + (size_t)r * n * D;
    double* gbeta = bp.gbeta + (size_t)r * E * n;
    double* gell = bp.gell + (size_t)r * E * D;
    for (int e = tid; e < n * D; e += nt) {
        const int nn = e / D, d = e % D;
        double v = 0.0;
        for (int tk = 0; tk < B.ntask; ++tk) v += wsr[B.Tz + ((size_t)tk * np + nn) * MAXD + d];
        gX[e] = bp.accumulate ? gX[e] + v : v;
    }
    for (int e = tid; e < E * n; e += nt) {
        const int a = e / n, nn = e % n;
        double v = wsr[B.Tb + (size_t)a * np + nn];
        for (int b = 0; b < E; ++b) v += wsr[B.Tb + (size_t)(E + a * E + b) * np + nn];
        gbeta[e] = bp.accumulate ? gbeta[e] + v : v;
    }
    for (int e = tid; e < E * D; e += nt) {
        const int a = e / D, d = e % D;
        double gp_ = 0.0;
        for (int b = 0; b < E; ++b) {
            gp_ += wsr[B.Tpa + (size_t)(E + a * E + b) * MAXD + d];      // row side of (a,b) + delta share
            gp_ += wsr[B.Tpb + (size_t)(E + b * E + a) * MAXD + d];      // delta share of (b,a)
        }
        const double l = ell[a * D + d];
        const double v = -2.0 * gp_ / (l * l * l) + 2.0 * l * wsr[B.Tpa + (size_t)a * MAXD + d];
        gell[e] = bp.accumulate ? gell[e] + v : v;
    }
}

// finish + reduce in ONE launch: one CTA per task; the last CTA of a restart to arrive sums the task partials (fixed
// task order: deterministic whichever CTA that is) -- one dependent kernel less on the serial path of the reverse sweep
template <int DP>
__global__ void __launch_bounds__(128, 2) mm_bfinish_kernel(MMBwdParams bp) {
    PDL_ENTRY();
    const int r = blockIdx.y;
    mm_bfinish_task<DP>(bp, r, blockIdx.x);
    unsigned* cnt = reinterpret_cast<unsigned*>(bp.f.ws + (size_t)r * bp.B.per_r + bp.B.cnt);
    if (last_cta_arrives(cnt, gridDim.x)) mm_breduce_body(bp, r);
}

// -------------------------------------------------------------------------------------------------
// host
// -------------------------------------------------------------------------------------------------
template <int KS>
static int launch_btile(const MMBwdParams& bp, cudaStream_t st) {
    const size_t smem = mm_btile_smem_bytes(bp.B.F.np, bp.B.F.ldz);
    if (pilco_smem_optin<mm_btile_kernel<KS, false>, mm_btile_kernel<KS, true>>((int)mm_btile_smem_bytes(TILE_CM, 20)))
        return PILCO_ERR_LAUNCH;
    const int E = bp.f.gp.E;
    { const dim3 gb(bp.B.F.NB, bp.B.P2, bp.f.R); launch_pri(pilco_small_grid(gb), mm_btile_kernel<KS, false>, gb, dim3(256), smem, st, bp); }
    if (bp.f.gp.mode == 0 && bp.f.gp.iK != nullptr)
        { const dim3 gb(bp.B.F.NB, E, bp.f.R); launch_pri(pilco_small_grid(gb), mm_btile_kernel<KS, true>, gb, dim3(256), smem, st, bp); }
    return PILCO_OK;
}

int mm_backward_launch(MMBwdParams bp, cudaStream_t st) {
    const int E = bp.f.gp.E, R = bp.f.R, D = bp.f.gp.D;
    MMParams sp = bp.f;                       // setup in ordered/backward mode on the same workspace
    sp.L = bp.B.F; sp.bwd = 1; sp.oQ = bp.B.oQ; sp.oC = bp.B.oC; sp.oLd = bp.B.oLd;
    // per-restart stride of the setup arrays must be the backward stride
    sp.L.per_r = bp.B.per_r;
    ks_dispatch(D, [&](auto ks) { mm_setup_launch<4 * ks, true>(sp, st); });
    CUDA_LAUNCH_CHECK();
    const int rc = ks_dispatch(D, [&](auto ks) { return launch_btile<ks>(bp, st); });
    if (rc) return rc;
    CUDA_LAUNCH_CHECK();
    const dim3 gf(E + E * E, R);
    ks_dispatch(D, [&](auto ks) { launch_hi(mm_bfinish_kernel<4 * ks>, gf, dim3(128), 0, st, bp); });
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

MMBwdParams mm_bwd_params(const pilco_gp_model* gp, int R, const double* m, long long m_rs, const double* s, long long s_rs,
                          const double* Mfwd, const double* gM, const double* gS, const double* gV,
                          double* gm, long long gm_rs, double* gs, long long gs_rs,
                          double* gX, double* gbeta, double* gell, int accumulate, double* ws) {
    MMBwdParams bp;
    bp.need_param = (gX && gbeta && gell) ? 1 : 0;
    bp.B = mm_bws_layout(gp->n, gp->D, gp->E, bp.need_param);
    bp.f = mm_params(gp, R, m, m_rs, s, s_rs, const_cast<double*>(Mfwd), nullptr, nullptr, nullptr, ws);
    bp.f.L = bp.B.F; bp.f.bwd = 1; bp.f.oQ = bp.B.oQ; bp.f.oC = bp.B.oC; bp.f.oLd = bp.B.oLd;
    bp.gM = gM; bp.gS = gS; bp.gV = gV;
    bp.gm = gm; bp.gs = gs; bp.gm_rs = gm_rs; bp.gs_rs = gs_rs;
    bp.gX = gX; bp.gbeta = gbeta; bp.gell = gell; bp.accumulate = accumulate;
    return bp;
}

extern "C" {

size_t pilco_mm_bwd_workspace_bytes(int n, int D, int E, int R, int need_param) {
    if (n < 1 || D < 1 || D > MAXD || E < 1 || E > MAXE || R < 1) return 0;
    return mm_bws_layout(n, D, E, need_param).per_r * (size_t)R * sizeof(double);
}

int pilco_mm_backward(const pilco_gp_model* gp, int R, const double* m, const double* s, const double* M,
                      const double* gM, const double* gS, const double* gV,
                      double* gm, double* gs, double* gX, double* gbeta, double* gell,
                      void* ws, size_t ws_bytes, pilco_stream_t stream) {
    int rc = mm_check_model(gp);
    if (rc) return rc;
    if (!m || !s || !M || !gM || !gS || !gV || !gm || !gs || !ws) return PILCO_ERR_NULL;
    if (R < 1) return PILCO_ERR_DIM;
    const int need_param = (gX && gbeta && gell) ? 1 : 0;
    if (ws_bytes < pilco_mm_bwd_workspace_bytes(gp->n, gp->D, gp->E, R, need_param)) return PILCO_ERR_WORKSPACE;
    if (((uintptr_t)ws) & 15) return PILCO_ERR_ALIGN;
    MMBwdParams bp = mm_bwd_params(gp, R, m, gp->D, s, (long long)gp->D * gp->D, M, gM, gS, gV,
                                   gm, gp->D, gs, (long long)gp->D * gp->D, gX, gbeta, gell, 0, (double*)ws);
    mm_bwd_zero_counters(bp.B, (double*)ws, R, (cudaStream_t)stream);
    return mm_backward_launch(bp, (cudaStream_t)stream);
}

}  // extern "C"

#ifdef PILCO_TILE_TIMING
// diagnostics build: phase stamps of the LAST backward tile launch (this translation unit's copy of g_tile_timing)
extern "C" int pilco_debug_btile_timing(long long* host_out, int n) {
    return (int)cudaMemcpyFromSymbol(host_out, g_tile_timing, sizeof(long long) * (size_t)n);
}
#endif
