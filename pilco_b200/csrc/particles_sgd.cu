// particles_sgd.cu -- the stochastic policy optimiser's device work (pilco_normals, pilco_adam_update; DESIGN.md
// section 32):
//   sgd_normals_kernel  one thread per pair of normals: Philox4x32-10 of (pair, stream, *iter) under the seed, two
//                       uniforms, Box-Muller.  *iter is read at run time, so a captured graph draws afresh per replay.
//   sgd_adam_kernel     one CTA per restart: the gradient row's status and fixed-order norm, the clip, the restart's
//                       step count and running products, the Adam step of each parameter and the trace row
//   sgd_tick_kernel     *iter += 1, after every restart's update has read it
// The arithmetic is sgd_math.cuh's, which the CPU tests compile for the host.  Deterministic (no atomics), no host
// synchronisation.
#include "common.cuh"
#include "sgd_math.cuh"

#define SGD_NTHREADS 256
#define SGD_MAX_GRID 8192

// grid-stride over the n / 2 (rounded up) pairs; element 2j + 1 of the last pair is not written when n is odd
__global__ void __launch_bounds__(SGD_NTHREADS) sgd_normals_kernel(unsigned long long seed, unsigned stream_id,
                                                                   const long long* iter, long long n, double* out) {
    PDL_ENTRY();
    const uint32_t it = (uint32_t)*iter;
    const long long pairs = (n + 1) >> 1;
    for (long long j = (long long)blockIdx.x * SGD_NTHREADS + threadIdx.x; j < pairs;
         j += (long long)gridDim.x * SGD_NTHREADS) {
        double u1, u2, z0, z1;
        sgd_pair_uniforms(seed, stream_id, it, (uint64_t)j, &u1, &u2);
        sgd_box_muller(u1, u2, &z0, &z1);
        out[2 * j] = z0;
        if (2 * j + 1 < n) out[2 * j + 1] = z1;
    }
}

struct AdamDev {
    int R, n, ld_theta, ld_packed, trace_rows;
    double lr, b1, b2, eps, max_norm;
    double* theta; const double* packed; double* m; double* v;
    long long* t; double* b1t; double* b2t; const long long* iter; double* trace; int* ok;
};

// grid R, SGD_LANES threads: restart blockIdx.x
__global__ void __launch_bounds__(SGD_LANES) sgd_adam_kernel(AdamDev a) {
    PDL_ENTRY();
    __shared__ double red[SGD_LANES];
    const int r = blockIdx.x, l = threadIdx.x;
    const double* row = a.packed + (size_t)r * a.ld_packed;
    const double loss = row[0], status = row[1];
    const double* g = row + 2;
    const long long k = *a.iter;
    const double b1t = a.b1t[r], b2t = a.b2t[r];       // read before thread 0 writes them below
    bool fin;
    red[l] = sgd_lane_sumsq(g, a.n, l, &fin);
    const bool all_finite = __syncthreads_and(fin) != 0;
    for (int half = SGD_LANES / 2; half > 0; half >>= 1) {
        if (l < half) sgd_tree_step(red, l, half);
        __syncthreads();
    }
    const bool ok = status == 0.0 && isfinite(loss) && all_finite;
    if (ok) {
        const double scale = sgd_clip_scale(red[0], a.max_norm);
        const double nb1t = sgd_mul(b1t, a.b1), nb2t = sgd_mul(b2t, a.b2);
        double* th = a.theta + (size_t)r * a.ld_theta;
        double* m = a.m + (size_t)r * a.n;
        double* v = a.v + (size_t)r * a.n;
        for (int i = l; i < a.n; i += SGD_LANES)
            sgd_adam_elem(g[i], scale, a.lr, a.b1, a.b2, a.eps, nb1t, nb2t, m + i, v + i, th + i);
        if (l == 0) {
            a.t[r] += 1;
            a.b1t[r] = nb1t;
            a.b2t[r] = nb2t;
        }
    }
    if (l == 0 && k >= 0 && k < a.trace_rows) {
        a.trace[(size_t)k * a.R + r] = -loss;
        a.ok[(size_t)k * a.R + r] = ok;
    }
}

__global__ void sgd_tick_kernel(long long* iter) {
    PDL_ENTRY();
    *iter += 1;
}

extern "C" {

int pilco_normals(unsigned long long seed, unsigned stream_id, const long long* iter, long long n, double* out,
                  pilco_stream_t stream) {
    if (!iter || !out) return PILCO_ERR_NULL;
    if (n < 0) return PILCO_ERR_DIM;
    if (n == 0) return PILCO_OK;
    const long long blocks = ((n + 1) / 2 + SGD_NTHREADS - 1) / SGD_NTHREADS;
    launch_hi(sgd_normals_kernel, dim3((unsigned)(blocks < SGD_MAX_GRID ? blocks : SGD_MAX_GRID)), dim3(SGD_NTHREADS),
              0, (cudaStream_t)stream, seed, stream_id, iter, n, out);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int pilco_adam_update(const pilco_adam* a, pilco_stream_t stream) {
    if (!a || !a->theta || !a->packed || !a->m || !a->v || !a->t || !a->b1t || !a->b2t || !a->iter)
        return PILCO_ERR_NULL;
    if (a->trace_rows > 0 && (!a->trace || !a->ok)) return PILCO_ERR_NULL;
    if (a->R < 1 || a->n < 1 || a->ld_theta < a->n || a->ld_packed < a->n + 2 || a->trace_rows < 0)
        return PILCO_ERR_DIM;
    if (!(a->lr > 0.0) || !isfinite(a->lr) || !(a->b1 >= 0.0 && a->b1 < 1.0) || !(a->b2 >= 0.0 && a->b2 < 1.0) ||
        !(a->eps > 0.0) || !(a->max_norm >= 0.0))
        return PILCO_ERR_DIM;
    AdamDev d;
    d.R = a->R; d.n = a->n; d.ld_theta = a->ld_theta; d.ld_packed = a->ld_packed; d.trace_rows = a->trace_rows;
    d.lr = a->lr; d.b1 = a->b1; d.b2 = a->b2; d.eps = a->eps; d.max_norm = a->max_norm;
    d.theta = a->theta; d.packed = a->packed; d.m = a->m; d.v = a->v;
    d.t = a->t; d.b1t = a->b1t; d.b2t = a->b2t; d.iter = a->iter; d.trace = a->trace; d.ok = a->ok;
    cudaStream_t st = (cudaStream_t)stream;
    launch_hi(sgd_adam_kernel, dim3(a->R), dim3(SGD_LANES), 0, st, d);
    CUDA_LAUNCH_CHECK();
    launch_hi(sgd_tick_kernel, dim3(1), dim3(1), 0, st, a->iter);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

}  // extern "C"
