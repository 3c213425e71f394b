// common.cuh -- shared device helpers for the PILCO engine (sm_90a).
//
// Small dense linear algebra on D<=16 matrices held in shared memory (one warp cooperates),
// the table-driven fp64 exp used by the tile kernels, DMMA wrappers, TMA bulk-copy wrappers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "../../include/pilco_b200.h"

#define PILCO_OK              0
#define PILCO_ERR_NULL       -1
#define PILCO_ERR_DIM        -2
#define PILCO_ERR_WORKSPACE  -3
#define PILCO_ERR_ALIGN      -4
#define PILCO_ERR_LAUNCH     -5
#define PILCO_ERR_UNSUPPORTED -6

#define MAXD PILCO_MAX_D
#define MAXE PILCO_MAX_E
#define SLD  17                 // leading dimension of small smem matrices (odd -> conflict-light)
#define PILCO_MAX_SMEM_OPTIN (227 * 1024)   // dynamic shared memory a CTA can opt in to on sm_90
#define NEG_PAD (-1.0e9)        // (scaled) exponent of padded rows/cols: exp_scaled() clamps it to ~1e-304

#define CUDA_LAUNCH_CHECK() do { cudaError_t e__ = cudaGetLastError(); if (e__ != cudaSuccess) return PILCO_ERR_LAUNCH; } while (0)

static inline __host__ __device__ int pad64(int n) { return (n + 63) & ~63; }
// reward kinds: the *_SA ones are evaluated on the joint state-action Gaussian / point (dimension D), the others on
// the state (dimension Ds); the exponential ones carry a target t
static inline __host__ __device__ bool reward_on_joint(int kind) { return kind == PILCO_REWARD_EXP_SA || kind == PILCO_REWARD_LINEAR_SA; }
static inline bool reward_kind_known(int kind) { return kind >= PILCO_REWARD_EXP && kind <= PILCO_REWARD_LINEAR_SA; }
static inline bool reward_needs_t(int kind) { return kind == PILCO_REWARD_EXP || kind == PILCO_REWARD_EXP_SA; }
// row stride (in doubles) of zeta/U rows: multiple of 4 (DMMA k-step) and == 4 or 12 (mod 16) so
// that the 8-column x 4-k B-fragment read is shared-memory bank-conflict free.
static inline __host__ __device__ int ldz_of(int D) { return D <= 4 ? 4 : (D <= 12 ? 12 : 20); }
static inline __host__ __device__ int ksteps_of(int D) { return (D + 3) / 4; }
static inline __host__ __device__ int npairs_of(int E) { return E * (E + 1) / 2; }

// unordered pair index q <-> (a,b), a<=b, b-major: q = b(b+1)/2 + a
static inline __host__ __device__ void pair_decode(int q, int& a, int& b) {
    int bb = 0;
    while ((bb + 1) * (bb + 2) / 2 <= q) ++bb;
    b = bb; a = q - bb * (bb + 1) / 2;
}
static inline __host__ __device__ int pair_index(int a, int b) { return a <= b ? b * (b + 1) / 2 + a : a * (a + 1) / 2 + b; }

#ifdef __CUDACC__

// ---------------------------------------------------------------------------------------------
// warp helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide sum of `cnt` values per thread-private array `vals` -> result in smem out[0..cnt)
// (valid for all threads after the trailing __syncthreads).  red must hold cnt*nwarps doubles.
template <int MAXCNT>
__device__ __forceinline__ void block_sum(double* vals, int cnt, double* red, double* out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int c = 0; c < cnt; ++c) {
        double v = warp_sum(vals[c]);
        if (lane == 0) red[c * nw + warp] = v;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < cnt; c += blockDim.x) {
        double v = 0.0;
        for (int w = 0; w < nw; ++w) v += red[c * nw + w];     // fixed order: deterministic
        out[c] = v;
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// small dense linear algebra, one warp, matrices in shared memory (row-major, leading dim SLD)
// ---------------------------------------------------------------------------------------------
// In-place lower Cholesky of the SPD matrix A[D][D] (only the lower triangle is referenced/written).
// invd[j] = 1/L[j][j].  Returns false (to all lanes) if a pivot is not positive.
__device__ __forceinline__ bool chol_warp(double* A, double* invd, int D, int lane) {
    bool ok = true;
    for (int j = 0; j < D; ++j) {
        double d = A[j * SLD + j];
        if (!(d > 0.0)) { ok = false; d = 1.0; }
        const double piv = sqrt(d);
        const double ip = 1.0 / piv;
        __syncwarp();
        if (lane == 0) { A[j * SLD + j] = piv; invd[j] = ip; }
        for (int i = j + 1 + lane; i < D; i += 32) A[i * SLD + j] *= ip;
        __syncwarp();
        // trailing update: entries (i,k), j<k<=i<D, flattened over lanes
        const int rem = D - j - 1;
        const int cnt = rem * (rem + 1) / 2;
        for (int e = lane; e < cnt; e += 32) {
            int ii = 0;
            while ((ii + 1) * (ii + 2) / 2 <= e) ++ii;
            const int kk = e - ii * (ii + 1) / 2;
            const int i = j + 1 + ii, k = j + 1 + kk;
            A[i * SLD + k] -= A[i * SLD + j] * A[k * SLD + j];
        }
        __syncwarp();
    }
    return ok;
}

// Solve (L L^T) Y = B for ncols right-hand sides, B/Y in smem [D][SLD] (in place), lane per column.
__device__ __forceinline__ void chol_solve_warp(const double* L, const double* invd, double* B,
                                                int D, int ncols, int lane) {
    for (int c = lane; c < ncols; c += 32) {
        for (int i = 0; i < D; ++i) {                   // forward: L y = b
            double v = B[i * SLD + c];
            for (int k = 0; k < i; ++k) v -= L[i * SLD + k] * B[k * SLD + c];
            B[i * SLD + c] = v * invd[i];
        }
        for (int i = D - 1; i >= 0; --i) {              // backward: L^T x = y
            double v = B[i * SLD + c];
            for (int k = i + 1; k < D; ++k) v -= L[k * SLD + i] * B[k * SLD + c];
            B[i * SLD + c] = v * invd[i];
        }
    }
    __syncwarp();
}

// log det of the factored matrix: 2 * sum log L_ii  (all lanes get the value)
__device__ __forceinline__ double chol_logdet(const double* invd, int D) {
    double acc = 0.0;
    for (int j = 0; j < D; ++j) acc -= log(invd[j]);
    return 2.0 * acc;
}

// LU with partial pivoting of A[D][D] in smem (in place), perm[D] row permutation, returns det
// sign * prod(diag) through *det.  One warp.
__device__ __forceinline__ void lu_warp(double* A, int* perm, int D, int lane, double* det) {
    double dsign = 1.0;
    for (int i = lane; i < D; i += 32) perm[i] = i;
    __syncwarp();
    for (int j = 0; j < D; ++j) {
        // pivot search (all lanes redundantly; D<=16)
        int p = j; double best = fabs(A[j * SLD + j]);
        for (int i = j + 1; i < D; ++i) { double v = fabs(A[i * SLD + j]); if (v > best) { best = v; p = i; } }
        __syncwarp();
        if (p != j) {
            for (int k = lane; k < D; k += 32) { double t = A[j * SLD + k]; A[j * SLD + k] = A[p * SLD + k]; A[p * SLD + k] = t; }
            if (lane == 0) { int t = perm[j]; perm[j] = perm[p]; perm[p] = t; }
            dsign = -dsign;
        }
        __syncwarp();
        const double ip = 1.0 / A[j * SLD + j];
        __syncwarp();
        for (int i = j + 1 + lane; i < D; i += 32) A[i * SLD + j] *= ip;
        __syncwarp();
        const int rem = D - j - 1;
        for (int e = lane; e < rem * rem; e += 32) {
            const int i = j + 1 + e / rem, k = j + 1 + e % rem;
            A[i * SLD + k] -= A[i * SLD + j] * A[j * SLD + k];
        }
        __syncwarp();
    }
    double d = dsign;
    for (int j = 0; j < D; ++j) d *= A[j * SLD + j];
    *det = d;
}

// Solve A X = B given LU (perm applied to B rows first); B in smem [D][SLD] holds the UNPERMUTED rhs,
// result written to Xo [D][SLD].  lane per column.
__device__ __forceinline__ void lu_solve_warp(const double* LU, const int* perm, const double* B, double* Xo,
                                              int D, int ncols, int lane) {
    for (int c = lane; c < ncols; c += 32) {
        for (int i = 0; i < D; ++i) {
            double v = B[perm[i] * SLD + c];
            for (int k = 0; k < i; ++k) v -= LU[i * SLD + k] * Xo[k * SLD + c];
            Xo[i * SLD + c] = v;
        }
        for (int i = D - 1; i >= 0; --i) {
            double v = Xo[i * SLD + c];
            for (int k = i + 1; k < D; ++k) v -= LU[i * SLD + k] * Xo[k * SLD + c];
            Xo[i * SLD + c] = v / LU[i * SLD + i];
        }
    }
    __syncwarp();
}

// ---------------------------------------------------------------------------------------------
// fp64 exp for the tile kernels: x = (k*64 + j) ln2/64 + r,  exp(x) = 2^k * T[j] * (1 + expm1(r)).
// |r| <= ln2/128 so a degree-5 expm1 polynomial is exact to < 1e-16 relative.  10 fp64-pipe
// instructions + one shared-memory table read; arguments below -700 are clamped (result ~1e-304).
// ---------------------------------------------------------------------------------------------
#include "exp_table.cuh"                   // EXP_TAB, EXP_SC, exp_scaled / exp_shifted / exp_row_split

// table T[j] = 2^(j/EXP_TAB), correctly rounded (scripts/gen_exp_table.py), compiled into the library: no run-time
// upload, no per-device state, so every entry point is CUDA-graph capturable from its first call
// (one copy per translation unit: the library is built without relocatable device code)
static __device__ __align__(16) const double g_exp_tab[EXP_TAB_DOUBLES] = {
#ifdef PILCO_EXP256
#include "exp_table_data256x16.inc"
#else
#include "exp_table_data.inc"
#endif
};
#define PILCO_MAX_DEVICES 64
static inline int pilco_current_device() {
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess || d < 0) d = 0;
    return d < PILCO_MAX_DEVICES ? d : PILCO_MAX_DEVICES - 1;
}
// SMs of the current device (cached per device): the launch heuristics size grids against the machine
static inline int pilco_sm_count() {
    static int count[PILCO_MAX_DEVICES] = {0};
    int& c = count[pilco_current_device()];
    if (c == 0) {
        int d = 0, v = 0;
        cudaGetDevice(&d);
        c = (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d) == cudaSuccess && v > 0) ? v : 132;
    }
    return c;
}

// ---------------------------------------------------------------------------------------------
// Launch priorities.  A rollout step is a chain of ~15 small latency-bound kernels around one (or two) big tile
// kernels; several sub-batches run on parallel streams so that one's chain overlaps another's tile pass.  The block
// scheduler dispatches grids of EQUAL priority in arrival order, so a 4-CTA glue kernel queues behind every not yet
// dispatched tile CTA of the other streams.  Glue kernels are therefore launched with the device's highest
// priority (cudaLaunchAttributePriority; kept by graph capture): their CTAs take the next free slot.
// PILCO_NO_PRIORITY=1 disables (A/B tuning switch).
// ---------------------------------------------------------------------------------------------
#include <stdlib.h>
#include <type_traits>
#include <utility>
static inline int pilco_hi_priority() {
    static int hi = 0x7fffffff;
    if (hi == 0x7fffffff) {
        int least = 0, greatest = 0;
        const char* e = getenv("PILCO_NO_PRIORITY");
        if (e && e[0] == '1') hi = 0;
        else { cudaDeviceGetStreamPriorityRange(&least, &greatest); hi = greatest; }
    }
    return hi;
}
#ifdef __CUDACC__
// Programmatic dependent launch: every kernel launched through launch_pri starts with pdl_wait() (griddepcontrol.wait:
// returns once the preceding grid in the stream has completed and its memory is visible) followed by pdl_trigger()
// (lets the NEXT grid's CTAs be scheduled early; they park in their own pdl_wait).  With the stream-serialisation
// attribute the launch latency and grid drain/fill gaps between the ~15 dependent kernels of a rollout step overlap
// instead of adding up.  Stream capture turns these into programmatic graph edges.
// The early-scheduled CTAs of the dependents hold SM resources the tile kernels of the other sub-batches could use, so
// it is OFF by default; PILCO_PDL=1 enables it (the device-side instructions are no-ops without the attribute).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#define PDL_ENTRY() do { pdl_wait(); pdl_trigger(); } while (0)
static inline int pilco_use_pdl() {
    static int use = -1;
    if (use < 0) { const char* e = getenv("PILCO_PDL"); use = (e && e[0] == '1') ? 1 : 0; }
    return use;
}
template <typename... KArgs, typename... Args>
static inline void launch_pri(bool hi, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributePriority;
    at[0].val.priority = hi ? pilco_hi_priority() : 0;
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pilco_use_pdl() ? 2 : 1;
    cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}
template <typename... KArgs, typename... Args>
static inline void launch_hi(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    launch_pri(true, kern, grid, block, smem, st, std::forward<Args>(args)...);
}
// "Last CTA" pattern: fold a small per-group follow-up kernel into the kernel that produces its inputs.  Returns true
// (to every thread) in exactly one CTA of the `count` CTAs sharing `counter`: the last one to arrive, which then sees
// every global write the others made before arriving.  The winner resets the counter (self-cleaning; the counter
// array must be zero before the first use).  Results stay deterministic as long as the follow-up work does not
// depend on WHICH CTA runs it.
__device__ __forceinline__ bool last_cta_arrives(unsigned* counter, unsigned count) {
    __shared__ int s_last_flag;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned prev = atomicAdd(counter, 1u);
        s_last_flag = (prev + 1 == count);
        if (s_last_flag) *counter = 0;
    }
    __syncthreads();
    const bool last = s_last_flag != 0;
    if (last) __threadfence();
    return last;
}

// tile-type kernels: "glue" (high priority) while the whole grid fits the machine once, bulk work otherwise
static inline bool pilco_small_grid(dim3 g) { return (long long)g.x * g.y * g.z < 2LL * pilco_sm_count(); }

// Calls f(std::integral_constant<int, KS>()) with the moment-match kernels' k-step count KS = ksteps_of(D) (1..4; 4
// beyond): the one map from a model's D to the template KS (or DP = 4 KS) the host launches.
template <class F>
static inline decltype(auto) ks_dispatch(int D, F&& f) {
    const int ks = ksteps_of(D);
    if (ks == 1) return f(std::integral_constant<int, 1>());
    if (ks == 2) return f(std::integral_constant<int, 2>());
    if (ks == 3) return f(std::integral_constant<int, 3>());
    return f(std::integral_constant<int, 4>());
}

// Opts the kernels Ks in to `bytes` of dynamic shared memory, in order, once per device (function attributes are per
// device; one flag per instantiation).  PILCO_ERR_LAUNCH if an attribute call fails.
template <auto... Ks>
static inline int pilco_smem_optin(int bytes) {
    static bool configured[PILCO_MAX_DEVICES] = {false};
    bool& done = configured[pilco_current_device()];
    if (!done) {
        if ((... || (cudaFuncSetAttribute(Ks, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess)))
            return PILCO_ERR_LAUNCH;
        done = true;
    }
    return PILCO_OK;
}
#endif

__device__ __forceinline__ void exp_table_init(double* tab) {
    for (int j = threadIdx.x; j < EXP_TAB_DOUBLES; j += blockDim.x) tab[j] = g_exp_tab[j];
}

// (exp_scaled, exp_shifted, exp_row_split: exp_table.cuh -- shared with the host test build)

// ---------------------------------------------------------------------------------------------
// DMMA: D(8x8) = A(8x4) * B(4x8) + C, fp64 (mma.sync: wgmma has no f64 kind).
// lane = 4*g + t:  a = A[g][t],  b = B[t][g],  c0/c1 = C[g][2t], C[g][2t+1].
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// ---------------------------------------------------------------------------------------------
// Hopper's native fp64 MMA shapes: D(16x8) = A(16xK) * B(Kx8) + C, K = 4, 8, 16 (SASS DMMA.16x8x4 / 16x8x8 / 16x8x16).
// lane = 4*g + t:  a[2i] = A[g][t + 4i],  a[2i+1] = A[g + 8][t + 4i],  b[i] = B[t + 4i][g],
//                  c[0], c[1] = C[g][2t], C[g][2t+1],  c[2], c[3] = C[g + 8][2t], C[g + 8][2t+1].
// Two 8x8x4 problems on row octets that share their B operand are ONE 16x8x4 problem: A rows 0-7 are the first octet's
// A fragment, rows 8-15 the second's, and the C fragment is the two octets' C fragments side by side.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void dmma1684(double (&c)[4], double a0, double a1, double b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a0), "d"(a1), "d"(b));
}
__device__ __forceinline__ void dmma1688(double (&c)[4], const double (&a)[4], double b0, double b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b0), "d"(b1));
}
__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                   "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// C(16x8) += A(16 x 4KS) B(4KS x 8) with the A fragment af[2ks + o] = A[8o + g][4ks + t] (two row octets, k-step ks)
// and the B fragment bf[ks] = B[4ks + t][g]: one MMA per K chunk, K = 4KS on Hopper's 16x8 shapes -- KS = 3 as
// 16x8x8 + 16x8x4 (PILCO_M16_K16PAD: one 16x8x16 whose fourth k-step has a zero A fragment; the B operand of that
// k-step repeats bf[2], finite, so the product adds exact zeros).
template <int KS>
__device__ __forceinline__ void mma16_k(double (&c)[4], const double (&af)[2 * KS], const double (&bf)[KS]) {
    if constexpr (KS == 1) {
        dmma1684(c, af[0], af[1], bf[0]);
    } else if constexpr (KS == 2) {
        dmma1688(c, af, bf[0], bf[1]);
    } else if constexpr (KS == 3) {
#ifdef PILCO_M16_K16PAD
        const double a8[8] = {af[0], af[1], af[2], af[3], af[4], af[5], 0.0, 0.0};
        const double b4[4] = {bf[0], bf[1], bf[2], bf[2]};
        dmma16816(c, a8, b4);
#else
        const double a4[4] = {af[0], af[1], af[2], af[3]};
        dmma1688(c, a4, bf[0], bf[1]);
        dmma1684(c, af[4], af[5], bf[2]);
#endif
    } else {
        static_assert(KS == 4, "K = 4 KS <= 16");
        const double b4[4] = {bf[0], bf[1], bf[2], bf[3]};
        dmma16816(c, af, b4);
    }
}

// ---------------------------------------------------------------------------------------------
// TMA bulk copy (1-D cp.async.bulk, SASS UBLKCP) global -> shared, completion on an mbarrier.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, unsigned parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
    while (!mbar_try_wait(bar, parity)) { }
}
// bytes must be a multiple of 16; both addresses 16-byte aligned
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                 :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

#endif  // __CUDACC__
