// fp64_mix.cu -- stand-alone microbenchmarks of the fp64 issue path on sm_90a: what does the tile kernels' instruction
// mix (DMMA.8x8x4 + DADD/DFMA/DMUL + integer + LDS) cost per warp, and which restructurings of the inner loop pay.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -o scripts/ubench/fp64_mix scripts/ubench/fp64_mix.cu
//   scripts/ubench/fp64_mix            (prints one line per pattern x occupancy)
//
// Every pattern runs ONE wave of (SMs x bpsm) CTAs of 256 threads (bpsm x 2 warps per SM sub-partition); elapsed SM cycles
// are read with clock64() in CTA 0.  `cyc/it` = elapsed cycles / (iterations x warps per sub-partition): the sub-partition
// cycles one warp-iteration costs at that occupancy.  `ideal` = 17 x DMMA + 2 x fp64 instructions of the iteration
// (fp64 pipe time at the peak rates measured on an H100 SXM at 1980 MHz: DMMA.8x8x4 31.7 TFLOP/s = 17 cycles per warp
// and sub-partition, DFMA / DADD / DMUL 2 cycles).  Diagnostics only: not part of the library.
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "../../pilco_b200/csrc/common.cuh"

#define NCOL 320
#define LDZ 12
#define KS 3

struct Smem {
    double sZ[NCOL * LDZ];
    double sBq[NCOL];
    double sBe[NCOL];
    double tab[EXP_TAB_DOUBLES];
};

__device__ __forceinline__ void fill_smem(Smem& s) {
    for (int i = threadIdx.x; i < NCOL * LDZ; i += blockDim.x) s.sZ[i] = 0.01 * ((i * 37) % 101 - 50);
    for (int i = threadIdx.x; i < NCOL; i += blockDim.x) { s.sBq[i] = -EXP_SC * (1.0 + 0.01 * (i % 97)); s.sBe[i] = 0.001 * ((i % 13) - 6); }
    exp_table_init(s.tab);
    __syncthreads();
}

// COST PROBE, not a valid exp: exp_shifted with the shift of the table offset dropped (one integer instruction fewer in the
// chain rounding -> offset -> LDS).  The idea behind it -- carry the integer field 3 bits up (magic 1.5*2^55) so that the
// byte offset is one LOP3 of the low word -- does not work: the mantissa field counts ulps, so with ulp 8 it holds
// round(x/8), not 8*round(x/8).  Kept because it measures what that one instruction costs (1.4 cycles per exp).
#define EXP_MAGIC8 (6755399441055744.0 * 8.0)
__device__ __forceinline__ double exp_shifted8(double c, double am, const double* __restrict__ tab) {
    const double t = c + am;
    const int lo = __double2loint(t), hi = __double2hiint(t);
    const double kd = t - am;
    const double r = c - kd;                                   // multiple-of-8 rounding: |r| <= 4
    double q = 5.169222938345892e-11 / 512.0;
    q = fma(q, r, 2.2909785199379098e-07 / 64.0);
    q = fma(q, r, 0.0006769015435155716 / 8.0);
    const double tj = *reinterpret_cast<const double*>(reinterpret_cast<const char*>(tab) + (lo & 0x1ff8));
    const double em1 = q * r;
    const double v = fma(tj, em1, tj);
    int k = (int)__funnelshift_r((unsigned)lo, (unsigned)hi, 13);
    k = max(k, -1008);
    int vh;
    asm("mad.lo.s32 %0, %1, 0x100000, %2;" : "=r"(vh) : "r"(k), "r"(__double2hiint(v)));
    return __hiloint2double(vh, __double2loint(v));
}

enum { P_DMMA_REG = 0, P_DMMA_LDS, P_DFMA, P_SEP, P_FINE, P_SEP_INT, P_EXP, P_EXP_NOLDS, P_EXP_NOINT, P_FULL, P_FULL8, P_FULL_SH8,
       P_FULL16, P_FULL_NOEXPINT, P_FULL_NOTAB, P_DADD, P_DFMA3, P_DFMA2, P_DMUL, P_SKEL, P_SKEL_ACC, P_FULL16_SH8, P_COUNT };
static const char* kNames[P_COUNT] = {
    "dmma_reg      12 DMMA, register operands",
    "dmma_lds      12 DMMA, B fragments + C from shared (as the kernel)",
    "dfma          64 DFMA, 8 chains",
    "sep           12 DMMA then 64 DFMA",
    "fine          (1 DMMA, 5-6 DFMA) x 12",
    "sep_int       12 DMMA then 64 DFMA + 64 integer ops",
    "exp           8 table exps + 8 DFMA accumulate (no DMMA)",
    "exp_nolds     ... table value from a register",
    "exp_noint     ... and no integer scaling/clamp",
    "full          the kernel's 4-tile group (12 LDS.64 + 8 LDS.128, 12 DMMA, 8 exp, 8 DFMA)",
    "full8         8-tile groups",
    "full_sh8      4-tile group, exp with ONE integer op fewer (cost probe only: not a valid exp, see exp_shifted8)",
    "full16        two row octets per warp share the B fragments (24 DMMA, 16 exp per group)",
    "full_noexpint 4-tile group, exp without integer scaling/clamp (wrong results; cost probe)",
    "full_notab    4-tile group, exp without the table gather (wrong results; cost probe)",
    "dadd          64 DADD a_i += b_i (distinct registers)",
    "dfma3         64 DFMA a_i = fma(a_i, b_i, c_i) (three distinct varying registers)",
    "dfma2         64 DFMA a_i = fma(a_i, b_i, const)",
    "dmul          64 DMUL a_i *= b_i",
    "skel          8 x the exp's 7 fp64 instructions only (no integer, no LDS)",
    "skel_acc      ... + DADD input + DFMA accumulate (9 per exp)",
    "full16_sh8    two row octets per warp + the one-op-fewer exp (cost probe)",
};
static const int kIdeal[P_COUNT] = {12 * 17, 12 * 17 + 16, 128, 332, 332, 332, 144, 144, 144, 332, 664, 332, 664, 332, 332, 128, 128, 128, 128, 112, 144, 664};

static double prop_clock_hz = 1.965e9;

template <int VAR>
__device__ __forceinline__ double exp_var(double c, double am, const double* tab) {
    if (VAR == 1) return exp_shifted8(c, am, tab);
    if (VAR == 2) {                                             // no integer scaling / clamp
        const double t = c + am;
        const int lo = __double2loint(t);
        const double kd = t - am;
        const double r = c - kd;
        EXP_POLY(q, r);
        const double tj = *reinterpret_cast<const double*>(reinterpret_cast<const char*>(tab) + EXP_TAB_OFFSET(lo));
        const double em1 = q * r;
        return fma(tj, em1, tj);
    }
    if (VAR == 3) {                                             // no table gather
        const double t = c + am;
        const int lo = __double2loint(t), hi = __double2hiint(t);
        const double kd = t - am;
        const double r = c - kd;
        EXP_POLY(q, r);
        const double tj = 1.25;
        const double em1 = q * r;
        const double v = fma(tj, em1, tj);
        int k = (int)__funnelshift_r((unsigned)lo, (unsigned)hi, EXP_SHIFT);
        k = max(k, -1008);
        int vh;
        asm("mad.lo.s32 %0, %1, 0x100000, %2;" : "=r"(vh) : "r"(k), "r"(__double2hiint(v)));
        return __hiloint2double(vh, __double2loint(v));
    }
    return exp_shifted(c, am, tab);
}

// the kernel's fast path: NT column tiles per group, exp variant VAR
template <int NT, int VAR>
__device__ __forceinline__ void sweep(const Smem& s, const double (&ua)[KS], double am, int g, int t, double& acc2) {
    for (int cg = 0; cg < NCOL; cg += 8 * NT) {
        double e[2 * NT];
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            const double2 bq = *reinterpret_cast<const double2*>(s.sBq + cg + 8 * j + 2 * t);
            e[2 * j] = bq.x; e[2 * j + 1] = bq.y;
        }
#pragma unroll
        for (int ks = 0; ks < KS; ++ks)
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                const double bf = s.sZ[(size_t)(cg + 8 * j + g) * LDZ + 4 * ks + t];
                dmma884(e[2 * j], e[2 * j + 1], ua[ks], bf);
            }
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            const double l0 = exp_var<VAR>(e[2 * j], am, s.tab), l1 = exp_var<VAR>(e[2 * j + 1], am, s.tab);
            const double2 bb = *reinterpret_cast<const double2*>(s.sBe + cg + 8 * j + 2 * t);
            acc2 = fma(bb.x, l0, acc2); acc2 = fma(bb.y, l1, acc2);
        }
    }
}

// two row octets per warp: the B fragment of a column tile feeds two DMMA
template <int VAR>
__device__ __forceinline__ void sweep16(const Smem& s, const double (&ua)[KS], const double (&ub)[KS], double am, double bm, int g, int t,
                                        double& acc2, double& acc3) {
    for (int cg = 0; cg < NCOL; cg += 32) {
        double e[8], f[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const double2 bq = *reinterpret_cast<const double2*>(s.sBq + cg + 8 * j + 2 * t);
            e[2 * j] = bq.x; e[2 * j + 1] = bq.y; f[2 * j] = bq.x; f[2 * j + 1] = bq.y;
        }
#pragma unroll
        for (int ks = 0; ks < KS; ++ks)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const double bf = s.sZ[(size_t)(cg + 8 * j + g) * LDZ + 4 * ks + t];
                dmma884(e[2 * j], e[2 * j + 1], ua[ks], bf);
                dmma884(f[2 * j], f[2 * j + 1], ub[ks], bf);
            }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const double2 bb = *reinterpret_cast<const double2*>(s.sBe + cg + 8 * j + 2 * t);
            const double l0 = exp_var<VAR>(e[2 * j], am, s.tab), l1 = exp_var<VAR>(e[2 * j + 1], am, s.tab);
            acc2 = fma(bb.x, l0, acc2); acc2 = fma(bb.y, l1, acc2);
            const double m0 = exp_var<VAR>(f[2 * j], bm, s.tab), m1 = exp_var<VAR>(f[2 * j + 1], bm, s.tab);
            acc3 = fma(bb.x, m0, acc3); acc3 = fma(bb.y, m1, acc3);
        }
    }
}

template <int PAT, int MINB>
__global__ void __launch_bounds__(256, MINB) pat_kernel(int iters, double* sink, long long* cyc) {
    extern __shared__ __align__(16) unsigned char raw[];
    Smem& s = *reinterpret_cast<Smem*>(raw);
    fill_smem(s);
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const double seed = 1.0 + 1e-9 * threadIdx.x;
    double a0 = seed, a1 = seed * 1.1, a2 = seed * 1.2, a3 = seed * 1.3, a4 = seed * 1.4, a5 = seed * 1.5, a6 = seed * 1.6, a7 = seed * 1.7;
    double c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0, c5 = 0, c6 = 0, c7 = 0;
    if (PAT == P_DADD || PAT == P_DFMA3 || PAT == P_DFMA2 || PAT == P_DMUL) {   // run-time values: real register operands
        c0 = sink[8]; c1 = sink[9]; c2 = sink[10]; c3 = sink[11]; c4 = sink[12]; c5 = sink[13]; c6 = sink[14]; c7 = sink[15];   // loaded: opaque to the compiler
    }
    int i0 = lane, i1 = lane + 1, i2 = lane + 2, i3 = lane + 3, i4 = lane + 4, i5 = lane + 5, i6 = lane + 6, i7 = lane + 7;
    const double m = 0.999999, b = 1e-7;
    double ua[KS], ub[KS];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) { ua[ks] = EXP_SC * 0.01 * ((lane * 7 + ks) % 11 - 5); ub[ks] = EXP_SC * 0.01 * ((lane * 5 + ks) % 13 - 6); }
    double am = EXP_MAGIC - 17.0, bm = EXP_MAGIC - 29.0, acc2 = 0.0, acc3 = 0.0;
    if (PAT == P_FULL_SH8 || PAT == P_FULL16_SH8) {
        bm = EXP_MAGIC8 - 29.0 * 8.0;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) ub[ks] *= 8.0;
        am = EXP_MAGIC8 - 17.0 * 8.0;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) ua[ks] *= 8.0;          // (sBq is not rescaled: only the cost matters here)
    }
    __syncthreads();
    const long long t0 = clock64();
    if ((PAT >= P_FULL && PAT <= P_FULL_NOTAB) || PAT == P_FULL16_SH8) {
        for (int it = 0; it < iters; ++it) {
            if (PAT == P_FULL) sweep<4, 0>(s, ua, am, g, t, acc2);
            if (PAT == P_FULL8) sweep<8, 0>(s, ua, am, g, t, acc2);
            if (PAT == P_FULL_SH8) sweep<4, 1>(s, ua, am, g, t, acc2);
            if (PAT == P_FULL16) sweep16<0>(s, ua, ub, am, bm, g, t, acc2, acc3);
            if (PAT == P_FULL16_SH8) sweep16<1>(s, ua, ub, am, bm, g, t, acc2, acc3);
            if (PAT == P_FULL_NOEXPINT) sweep<4, 2>(s, ua, am, g, t, acc2);
            if (PAT == P_FULL_NOTAB) sweep<4, 3>(s, ua, am, g, t, acc2);
            ua[0] += 1e-12;                                      // keep the sweeps distinct
        }
    } else {
        for (int it = 0; it < iters; ++it) {
            if (PAT == P_DMMA_REG) {
                dmma884(c0, c1, a0, a1); dmma884(c2, c3, a2, a3); dmma884(c4, c5, a4, a5); dmma884(c6, c7, a6, a7);
                dmma884(c0, c1, a1, a2); dmma884(c2, c3, a3, a4); dmma884(c4, c5, a5, a6); dmma884(c6, c7, a7, a0);
                dmma884(c0, c1, a2, a3); dmma884(c2, c3, a4, a5); dmma884(c4, c5, a6, a7); dmma884(c6, c7, a0, a1);
            }
            if (PAT == P_DMMA_LDS) {
                const int cg = (it * 32) % NCOL;
                double e[8];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const double2 bq = *reinterpret_cast<const double2*>(s.sBq + cg + 8 * j + 2 * t);
                    e[2 * j] = bq.x; e[2 * j + 1] = bq.y;
                }
#pragma unroll
                for (int ks = 0; ks < KS; ++ks)
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const double bf = s.sZ[(size_t)(cg + 8 * j + g) * LDZ + 4 * ks + t];
                        dmma884(e[2 * j], e[2 * j + 1], ua[ks], bf);
                    }
                c0 += e[0] + e[2] + e[4] + e[6]; c1 += e[1] + e[3] + e[5] + e[7];   // 8 DADD (counted in the note)
            }
            if (PAT == P_DFMA || PAT == P_SEP || PAT == P_SEP_INT) {
                if (PAT != P_DFMA) {
                    dmma884(c0, c1, a0, a1); dmma884(c2, c3, a2, a3); dmma884(c4, c5, a4, a5); dmma884(c6, c7, a6, a7);
                    dmma884(c0, c1, a1, a2); dmma884(c2, c3, a3, a4); dmma884(c4, c5, a5, a6); dmma884(c6, c7, a7, a0);
                    dmma884(c0, c1, a2, a3); dmma884(c2, c3, a4, a5); dmma884(c4, c5, a6, a7); dmma884(c6, c7, a0, a1);
                }
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    a0 = fma(a0, m, b); a1 = fma(a1, m, b); a2 = fma(a2, m, b); a3 = fma(a3, m, b);
                    a4 = fma(a4, m, b); a5 = fma(a5, m, b); a6 = fma(a6, m, b); a7 = fma(a7, m, b);
                    if (PAT == P_SEP_INT) {
                        i0 = (i0 ^ it) + 3; i1 = (i1 ^ it) + 5; i2 = (i2 ^ it) + 7; i3 = (i3 ^ it) + 9;   // 2 ops each
                    }
                }
            }
            if (PAT == P_DADD || PAT == P_DFMA3 || PAT == P_DFMA2 || PAT == P_DMUL) {
                // b_i = c0..c7 (distinct live registers, never written in this pattern)
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    if (PAT == P_DADD) { a0 += c0; a1 += c1; a2 += c2; a3 += c3; a4 += c4; a5 += c5; a6 += c6; a7 += c7; }
                    if (PAT == P_DFMA3) { a0 = fma(a0, c0, c1); a1 = fma(a1, c1, c2); a2 = fma(a2, c2, c3); a3 = fma(a3, c3, c4);
                                          a4 = fma(a4, c4, c5); a5 = fma(a5, c5, c6); a6 = fma(a6, c6, c7); a7 = fma(a7, c7, c0); }
                    if (PAT == P_DFMA2) { a0 = fma(a0, c0, b); a1 = fma(a1, c1, b); a2 = fma(a2, c2, b); a3 = fma(a3, c3, b);
                                          a4 = fma(a4, c4, b); a5 = fma(a5, c5, b); a6 = fma(a6, c6, b); a7 = fma(a7, c7, b); }
                    if (PAT == P_DMUL) { a0 *= c0; a1 *= c1; a2 *= c2; a3 *= c3; a4 *= c4; a5 *= c5; a6 *= c6; a7 *= c7; }
                }
            }
            if (PAT == P_SKEL || PAT == P_SKEL_ACC) {
                const double base = -EXP_SC * (2.0 + 1e-3 * (it & 1023));
#define SKEL(a, c) { const double x_ = PAT == P_SKEL_ACC ? base + a : a; const double t_ = x_ + am; const double kd_ = t_ - am; const double r_ = x_ - kd_; \
                     EXP_POLY(q_, r_); const double em_ = q_ * r_; const double v_ = fma(bm, em_, bm); \
                     if (PAT == P_SKEL_ACC) c = fma(b, v_, c); else a = v_; }
                SKEL(a0, c0) SKEL(a1, c1) SKEL(a2, c2) SKEL(a3, c3) SKEL(a4, c4) SKEL(a5, c5) SKEL(a6, c6) SKEL(a7, c7)
            }
            if (PAT == P_FINE) {
#define F5(x) a0 = fma(a0, m, b); a1 = fma(a1, m, b); a2 = fma(a2, m, b); a3 = fma(a3, m, b); a4 = fma(a4, m, b); x
                dmma884(c0, c1, a0, a1); F5(a5 = fma(a5, m, b);) dmma884(c2, c3, a2, a3); F5(a6 = fma(a6, m, b);)
                dmma884(c4, c5, a4, a5); F5(a7 = fma(a7, m, b);) dmma884(c6, c7, a6, a7); F5(a5 = fma(a5, m, b);)
                dmma884(c0, c1, a1, a2); F5(;) dmma884(c2, c3, a3, a4); F5(;) dmma884(c4, c5, a5, a6); F5(;) dmma884(c6, c7, a7, a0); F5(;)
                dmma884(c0, c1, a2, a3); F5(;) dmma884(c2, c3, a4, a5); F5(;) dmma884(c4, c5, a6, a7); F5(;) dmma884(c6, c7, a0, a1); F5(;)
            }
            if (PAT == P_EXP || PAT == P_EXP_NOLDS || PAT == P_EXP_NOINT) {
                // independent inputs every iteration (no chain through the exp): cost, not latency
                const double base = -EXP_SC * (2.0 + 1e-3 * (it & 1023));
                constexpr int V = PAT == P_EXP ? 0 : (PAT == P_EXP_NOLDS ? 3 : 2);
                c0 = fma(b, exp_var<V>(base + a0, am, s.tab), c0); c1 = fma(b, exp_var<V>(base + a1, am, s.tab), c1);
                c2 = fma(b, exp_var<V>(base + a2, am, s.tab), c2); c3 = fma(b, exp_var<V>(base + a3, am, s.tab), c3);
                c4 = fma(b, exp_var<V>(base + a4, am, s.tab), c4); c5 = fma(b, exp_var<V>(base + a5, am, s.tab), c5);
                c6 = fma(b, exp_var<V>(base + a6, am, s.tab), c6); c7 = fma(b, exp_var<V>(base + a7, am, s.tab), c7);
            }
        }
    }
    const long long t1 = clock64();
    if (blockIdx.x == 0 && threadIdx.x == 0) cyc[0] = t1 - t0;
    const double r = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7 + c0 + c1 + c2 + c3 + c4 + c5 + c6 + c7 + acc2 + acc3 +
                     (double)(i0 + i1 + i2 + i3 + i4 + i5 + i6 + i7);
    if (r == 123.456) sink[0] = r;
}

template <int PAT, int MINB>
static void run(int iters, double* sink, long long* cyc_dev, int nsm) {
    constexpr int bpsm = MINB;
    auto kern = pat_kernel<PAT, MINB>;
    // dynamic shared memory sized so that exactly `bpsm` CTAs fit an SM
    const int smem = ((227 * 1024) / bpsm - 1024) & ~1023;
    if (smem < (int)sizeof(Smem)) return;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    cudaFuncAttributes fa;
    cudaFuncGetAttributes(&fa, kern);
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 256, smem);
    if (occ != bpsm) { printf("%-14.14s bpsm=%d  skipped (occupancy %d, %d regs)\n", kNames[PAT], bpsm, occ, fa.numRegs); return; }
    const int sweeps = PAT >= P_FULL ? 1 : 1;
    (void)sweeps;
    long long cyc = 0;
    float ms = 0.f;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int rep = 0; rep < 2; ++rep) {
        cudaEventRecord(e0);
        kern<<<nsm * bpsm, 256, smem>>>(iters, sink, cyc_dev);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
    }
    cudaEventElapsedTime(&ms, e0, e1);
    cudaMemcpy(&cyc, cyc_dev, sizeof(cyc), cudaMemcpyDeviceToHost);
    cudaError_t err = cudaGetLastError();
    // warp-iterations per sub-partition: full patterns do NCOL/(8 NT) groups per `iteration`
    double groups = iters;
    if (PAT == P_FULL || PAT == P_FULL_SH8 || PAT == P_FULL16 || PAT == P_FULL_NOEXPINT || PAT == P_FULL_NOTAB || PAT == P_FULL16_SH8) groups = (double)iters * (NCOL / 32);
    if (PAT == P_FULL8) groups = (double)iters * (NCOL / 64);
    const double per_blk0 = (double)cyc / (groups * bpsm * 2);      // from CTA 0's own clock (== per when all CTAs are co-resident)
    const double per = (double)ms * 1e-3 * prop_clock_hz / (groups * bpsm * 2);
    printf("%-14.14s bpsm=%d warps/smsp=%2d regs=%3d  %8.3f ms  cyc/it %8.1f  ideal %4d  frac %.3f  (cta0 %.1f) %s\n", kNames[PAT], bpsm, bpsm * 2,
           fa.numRegs, ms, per, kIdeal[PAT], kIdeal[PAT] / per, per_blk0, err == cudaSuccess ? "" : cudaGetErrorString(err));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
}

template <int PAT>
static void run_all(double* sink, long long* cyc, int nsm) {
    const int iters = ((PAT >= P_FULL && PAT <= P_FULL_NOTAB) || PAT == P_FULL16_SH8) ? 400 : 4000;
    run<PAT, 1>(iters, sink, cyc, nsm); run<PAT, 2>(iters, sink, cyc, nsm); run<PAT, 3>(iters, sink, cyc, nsm);
    run<PAT, 4>(iters, sink, cyc, nsm); run<PAT, 5>(iters, sink, cyc, nsm);
    printf("   ^ %s\n", kNames[PAT]);
}

int main() {
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    printf("device %s, %d SMs, clock %d kHz\n", prop.name, prop.multiProcessorCount, prop.clockRate);
    double* sink; long long* cyc;
    cudaMalloc(&sink, 256);
    { double h[32]; for (int i = 0; i < 32; ++i) h[i] = 0.99999 + 1e-7 * i; cudaMemcpy(sink, h, sizeof(h), cudaMemcpyHostToDevice); } cudaMalloc(&cyc, 64);
    const int nsm = prop.multiProcessorCount;
    prop_clock_hz = prop.clockRate * 1e3;
    if (getenv("UBENCH_ALL")) {
        run_all<P_DMMA_REG>(sink, cyc, nsm); run_all<P_DMMA_LDS>(sink, cyc, nsm); run_all<P_DFMA>(sink, cyc, nsm); run_all<P_SEP>(sink, cyc, nsm);
        run_all<P_FINE>(sink, cyc, nsm); run_all<P_SEP_INT>(sink, cyc, nsm); run_all<P_EXP>(sink, cyc, nsm); run_all<P_EXP_NOLDS>(sink, cyc, nsm);
        run_all<P_EXP_NOINT>(sink, cyc, nsm); run_all<P_FULL8>(sink, cyc, nsm); run_all<P_FULL_NOEXPINT>(sink, cyc, nsm); run_all<P_FULL_NOTAB>(sink, cyc, nsm);
    }
    run_all<P_DFMA>(sink, cyc, nsm); run_all<P_DADD>(sink, cyc, nsm); run_all<P_DFMA3>(sink, cyc, nsm); run_all<P_DFMA2>(sink, cyc, nsm);
    run_all<P_DMUL>(sink, cyc, nsm); run_all<P_SKEL>(sink, cyc, nsm); run_all<P_SKEL_ACC>(sink, cyc, nsm);
    run_all<P_FULL>(sink, cyc, nsm); run_all<P_FULL_SH8>(sink, cyc, nsm); run_all<P_FULL16>(sink, cyc, nsm); run_all<P_FULL16_SH8>(sink, cyc, nsm);
    return 0;
}
