// particles_cem.cu -- the cross-entropy method's update on the device (pilco_cem_update, pilco_cem_draw; DESIGN.md
// section 31).  One iteration over K candidate action sequences cand [K,H,U] with their values is three kernels:
//   cem_rank_kernel   one CTA sorts the (value, index) pairs into rank order in shared memory (bitonic, no atomics),
//                     writes the order, the trace row and the best value so far
//   cem_refit_kernel  one thread per (t, u): the elites' mean and biased variance in rank order, the smoothed
//                     sampling distribution, and the best candidate's element when the best value rose
//   cem_draw_kernel   one thread per candidate element: the next candidates clip(mean + std xi) (row 0: clip(mean))
// The arithmetic is cem_math.cuh's, which the CPU tests compile for the host.  Deterministic, no host synchronisation.
#include "common.cuh"
#include "cem_math.cuh"

#define CEM_MAX_K    8192
#define CEM_MAX_HU   (1 << 24)
#define CEM_RTHREADS 1024

struct CemDev {
    int K, HU, ke;
    double alpha, lo, hi;
    const double* value; double* cand; const double* xi;
    double* mean; double* std;
    double* best_value; double* best; double* trace;
    int* order;                                         // [K] the rank order (workspace)
    int* improved;                                      // [1] this iteration raised the best value (workspace)
};

// grid 1, CEM_RTHREADS threads, N (a power of two >= K) x 12 bytes of dynamic shared memory.  Padding slots hold NaN
// with indices >= K, so they sort after every candidate.
__global__ void __launch_bounds__(CEM_RTHREADS) cem_rank_kernel(CemDev a, int N) {
    PDL_ENTRY();
    extern __shared__ double sv[];                      // [N] values, then [N] indices
    int* si = reinterpret_cast<int*>(sv + N);
    for (int i = threadIdx.x; i < N; i += CEM_RTHREADS) {
        sv[i] = i < a.K ? a.value[i] : __longlong_as_double(0x7ff8000000000000LL);
        si[i] = i;
    }
    __syncthreads();
    for (int k = 2; k <= N; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < N; i += CEM_RTHREADS) cem_bitonic_step(sv, si, i, j, k);
            __syncthreads();
        }
    for (int i = threadIdx.x; i < a.K; i += CEM_RTHREADS) a.order[i] = si[i];
    if (threadIdx.x == 0) {
        const double top = sv[0];
        double s = 0.0;
        for (int q = 0; q < a.ke; ++q) s = cem_add(s, sv[q]);
        if (a.trace) { a.trace[0] = top; a.trace[1] = s / a.ke; }
        const bool up = top > *a.best_value;            // strictly: a NaN or a tie keeps the earlier best
        if (up) *a.best_value = top;
        *a.improved = up;
    }
}

// grid ceil(HU / 128), 128 threads: element e of the sampling distribution (and of the best candidate)
__global__ void __launch_bounds__(128) cem_refit_kernel(CemDev a) {
    PDL_ENTRY();
    const int e = blockIdx.x * 128 + threadIdx.x;
    if (e >= a.HU) return;
    if (*a.improved) a.best[e] = a.cand[(size_t)a.order[0] * a.HU + e];
    double m = a.mean[e], s = a.std[e];
    cem_refit(a.cand, a.order, a.ke, (size_t)a.HU, (size_t)e, a.alpha, &m, &s);
    a.mean[e] = m;
    a.std[e] = s;
}

// grid ceil(K HU / 256), 256 threads: candidate element q = k HU + e
__global__ void __launch_bounds__(256) cem_draw_kernel(CemDev a) {
    PDL_ENTRY();
    const size_t q = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (q >= (size_t)a.K * a.HU) return;
    const int k = (int)(q / a.HU);
    const size_t e = q - (size_t)k * a.HU;
    a.cand[q] = cem_draw(k, a.mean[e], a.std[e], k ? a.xi[q] : 0.0, a.lo, a.hi);
}

// the bitonic sort's length: the least power of two >= K
static int cem_sort_len(int K) {
    int N = 1;
    while (N < K) N <<= 1;
    return N;
}

// Everything but the workspace, in this order: PILCO_ERR_NULL for c or a pointer the call reads or writes (the draw:
// cand, xi, mean, std; the update: value, cand, mean, std, best_value, best), then PILCO_ERR_DIM for K outside
// 1 .. 8192, H < 1, U < 1, H U > 2^24, lo >= hi (or a NaN bound), and for the update k_e outside 1 .. K or alpha
// outside [0, 1) (NaN included).
static int cem_check(const pilco_cem* c, bool update) {
    if (!c || !c->cand || !c->mean || !c->std) return PILCO_ERR_NULL;
    if (update ? (!c->value || !c->best_value || !c->best) : !c->xi) return PILCO_ERR_NULL;
    if (c->K < 1 || c->K > CEM_MAX_K || c->H < 1 || c->U < 1 || (long long)c->H * c->U > CEM_MAX_HU)
        return PILCO_ERR_DIM;
    if (!(c->lo < c->hi)) return PILCO_ERR_DIM;
    if (update && (c->n_elite < 1 || c->n_elite > c->K || !(c->alpha >= 0.0 && c->alpha < 1.0)))
        return PILCO_ERR_DIM;
    return PILCO_OK;
}

static CemDev cem_dev(const pilco_cem* c) {
    CemDev d;
    d.K = c->K; d.HU = c->H * c->U; d.ke = c->n_elite;
    d.alpha = c->alpha; d.lo = c->lo; d.hi = c->hi;
    d.value = c->value; d.cand = c->cand; d.xi = c->xi;
    d.mean = c->mean; d.std = c->std;
    d.best_value = c->best_value; d.best = c->best; d.trace = c->trace;
    d.order = nullptr; d.improved = nullptr;
    return d;
}

static int cem_draw_launch(cudaStream_t st, const CemDev& d) {
    const size_t n = (size_t)d.K * d.HU;
    launch_hi(cem_draw_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, d);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

extern "C" {

size_t pilco_cem_update_workspace_bytes(int K) {
    if (K < 1 || K > CEM_MAX_K) return 0;
    return ((size_t)(K + 1) * sizeof(int) + 15) / 16 * 16;
}

int pilco_cem_update(const pilco_cem* c, void* ws, size_t ws_bytes, pilco_stream_t stream) {
    if (const int rc = cem_check(c, true)) return rc;
    if (!ws) return PILCO_ERR_NULL;
    if ((uintptr_t)ws & 15) return PILCO_ERR_ALIGN;
    if (ws_bytes < pilco_cem_update_workspace_bytes(c->K)) return PILCO_ERR_WORKSPACE;
    if (const int rc = pilco_smem_optin<cem_rank_kernel>(CEM_MAX_K * 12)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    CemDev d = cem_dev(c);
    d.order = (int*)ws; d.improved = d.order + c->K;
    const int N = cem_sort_len(c->K);
    launch_hi(cem_rank_kernel, dim3(1), dim3(CEM_RTHREADS), (size_t)N * 12, st, d, N);
    CUDA_LAUNCH_CHECK();
    launch_hi(cem_refit_kernel, dim3((d.HU + 127) / 128), dim3(128), 0, st, d);
    CUDA_LAUNCH_CHECK();
    return c->xi ? cem_draw_launch(st, d) : PILCO_OK;
}

int pilco_cem_draw(const pilco_cem* c, pilco_stream_t stream) {
    if (const int rc = cem_check(c, false)) return rc;
    return cem_draw_launch((cudaStream_t)stream, cem_dev(c));
}

}  // extern "C"
