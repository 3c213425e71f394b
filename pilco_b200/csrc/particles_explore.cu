// particles_explore.cu -- PILCO's exploration objective in the particle rollouts (DESIGN.md section 24):
//   value[r] = (1/P) sum_p ret_p + b sum_t sigma_t,  sigma_t^2 = sum_k c_k^2 s_kt^2  (ADD-channel terms)
// with s_kt^2 the unbiased sample variance of term k's value over restart r's P particles at step t: the spread of the
// step's reward that the learnt model produces, the sampled counterpart of section 21's closed-form Var[r_t].
// Three kernels, each beside the existing launches (no existing kernel changes):
//   px_moments_kernel  once after the forward: the per-(restart, step, term) means and variances, sigma_t^2, sigma_t
//                      and the reverse sweep's table (mean_kt, P b c_k^2 / ((P-1) sigma_t))
//   px_bonus_kernel    at each reverse step t, after the step's VJP and before the step kernel: the bonus's cotangent
//                      sum_k a_kpt grad r_k into x_bar (state terms) or x~_bar_t (joint terms)
//   px_value_kernel    after the reduction: value[r] += b sum_t sigma_t
// The sums over a restart's particles are fixed-order (thread q takes p = q, q + 256, ..., then pg_block_sum), so a
// restart's statistics do not depend on R or on how the forward was chunked.
#include "particles.cuh"

// additive term k at the point x (global or shared memory) of width n: LINEAR(_SA) x' W, EXP(_SA) exp(-0.5 v' W v),
// v = x - t, in pt_reward_value's order (plain loops: a handful of registers, no indexed register arrays)
__device__ __forceinline__ double px_value(const pilco_reward_term& rt, const double* x, int n) {
    double acc = 0.0;
    if (rt.kind == PILCO_REWARD_LINEAR || rt.kind == PILCO_REWARD_LINEAR_SA) {
        for (int i = 0; i < n; ++i) acc = fma(x[i], rt.W[i], acc);
        return acc;
    }
    for (int i = 0; i < n; ++i) {
        double wy = 0.0;
        for (int k = 0; k < n; ++k) wy = fma(rt.W[i * n + k], x[k] - rt.t[k], wy);
        acc = fma(x[i] - rt.t[i], wy, acc);
    }
    return exp(-0.5 * acc);
}

// x~ = [phi(x), u] of one particle and step into xs (phi as pa_step_kernel forms it: sincospi of x / pi)
__device__ __forceinline__ void px_joint_point(const TrigMap& tm, const double* x, const double* u, int U, double* xs) {
    const int Dh = tm.Ds + tm.A, np = tm.np;
    for (int k = 0; k < Dh; ++k) {
        const int q = k - np;
        double f = x[q < 0 ? tm.pass[k] : tm.ang[q >> 1]];
        if (q >= 0) {
            double sn, cs;
            sincospi(f * PT_INV_PI, &sn, &cs);
            f = (q & 1) ? cs : sn;
        }
        xs[k] = f;
    }
    for (int j = 0; j < U; ++j) xs[Dh + j] = u[j];
}

// grid (H, R), 256 threads: step t = blockIdx.x of restart r = blockIdx.y.  One term at a time, two passes (mean, then
// squared deviations), each a fixed-order block sum; x~ is staged in a shared row per thread.
__global__ void __launch_bounds__(256) px_moments_kernel(PxMom a) {
    PDL_ENTRY();
    __shared__ double xs[256 * MAXD];
    __shared__ double red[8], out[1], km[8], kv[8];
    const int t = blockIdx.x, r = blockIdx.y, tid = threadIdx.x, P = a.P, H = a.H, U = a.U, E = a.tm.Ds;
    const int D = E + a.tm.A + U;
    const size_t r0 = (size_t)r * P;
    double* row = xs + tid * MAXD;
    for (int k = 0; k < a.n_rewards; ++k) {
        const pilco_reward_term& rt = a.rewards[k];
        if (rt.channel == PILCO_CHANNEL_MULT) {
            if (tid == 0) { km[k] = 0.0; kv[k] = 0.0; }
            continue;
        }
        const bool joint = reward_on_joint(rt.kind);
        auto value = [&](int p) -> double {
            const double* x = a.traj + ((r0 + p) * (H + 1) + t) * E;
            if (!joint) return px_value(rt, x, E);
            px_joint_point(a.tm, x, a.act + ((r0 + p) * H + t) * U, U, row);
            return px_value(rt, row, D);
        };
        double v[1] = {0.0};
        for (int p = tid; p < P; p += 256) v[0] += value(p);
        pg_block_sum<1>(v, red, out);
        const double mean = out[0] / P;
        v[0] = 0.0;
        for (int p = tid; p < P; p += 256) { const double d = value(p) - mean; v[0] = fma(d, d, v[0]); }
        pg_block_sum<1>(v, red, out);
        if (tid == 0) { km[k] = mean; kv[k] = out[0] / (P - 1); }
    }
    if (tid != 0) return;
    double m = 0.0, s2 = 0.0;
    for (int k = 0; k < a.n_rewards; ++k) {
        const double c = a.rewards[k].channel == PILCO_CHANNEL_MULT ? 0.0 : a.rewards[k].coef;
        m = fma(c, km[k], m);
        s2 = fma(c * c, kv[k], s2);
    }
    const double sd = s2 > 1e-12 ? sqrt(s2) : 0.0;      // section 21's floor: no gradient below it
    const size_t o = (size_t)r * H + t;
    if (a.step_mean) a.step_mean[o] = m;
    if (a.step_var) a.step_var[o] = s2;
    if (a.sd) a.sd[o] = sd;
    if (a.tab) {
        const double f = sd > 0.0 ? (double)P * a.b / ((double)(P - 1) * sd) : 0.0;
        double* tb = a.tab + o * a.n_rewards * 2;
        for (int k = 0; k < a.n_rewards; ++k) {
            const double c = a.rewards[k].channel == PILCO_CHANNEL_MULT ? 0.0 : a.rewards[k].coef;
            tb[2 * k] = km[k];
            tb[2 * k + 1] = f * (c * c);
        }
    }
}

// grid (ceil(P / 128), R), one thread per particle p of restart r = blockIdx.y at step t: x_bar (state terms, in E) or
// x~_bar_t (joint terms, all D columns) += a_kpt grad r_k, a_kpt = w_kt (r_kpt - mean_kt); the gradient of
// exp(-0.5 v' W v) is -value (W + W') v / 2, as pj_grad_kernel
__global__ void __launch_bounds__(PT_THREADS) px_bonus_kernel(PxBonus a) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x, r = blockIdx.y;
    if (p >= a.P) return;
    const int E = a.E, D = a.D, H = a.H, t = a.t, K = a.n_rewards;
    const size_t row = (size_t)r * a.P + p;
    const double* tb = a.tab + ((size_t)r * H + t) * K * 2;
    for (int k = 0; k < K; ++k) {
        const pilco_reward_term& rt = a.rewards[k];
        const double w = tb[2 * k + 1];
        if (rt.channel == PILCO_CHANNEL_MULT || w == 0.0) continue;
        const bool joint = reward_on_joint(rt.kind);
        const int n = joint ? D : E;
        const double* x = joint ? a.xh + row * D : a.traj + (row * (H + 1) + t) * E;
        double* g = joint ? a.gxt + row * D : a.gx + row * E;
        const double val = px_value(rt, x, n), c = w * (val - tb[2 * k]);
        if (rt.kind == PILCO_REWARD_LINEAR || rt.kind == PILCO_REWARD_LINEAR_SA) {
            for (int i = 0; i < n; ++i) g[i] = fma(c, rt.W[i], g[i]);
            continue;
        }
        const double f = -0.5 * c * val;
        for (int i = 0; i < n; ++i) {
            double wv = 0.0;
            for (int k2 = 0; k2 < n; ++k2) wv = fma(rt.W[i * n + k2] + rt.W[k2 * n + i], x[k2] - rt.t[k2], wv);
            g[i] = fma(f, wv, g[i]);
        }
    }
}

// one thread per restart: value[r] += b sum_t sd[r,t], the bonus summed in step order
__global__ void __launch_bounds__(128) px_value_kernel(int R, int H, double b, const double* sd, double* value) {
    PDL_ENTRY();
    const int r = blockIdx.x * 128 + threadIdx.x;
    if (r >= R) return;
    double s = 0.0;
    for (int t = 0; t < H; ++t) s += sd[(size_t)r * H + t];
    value[r] = fma(b, s, value[r]);
}

int px_moments_launch(cudaStream_t st, int R, const PxMom& a) {
    if (a.H == 0) return PILCO_OK;
    launch_hi(px_moments_kernel, dim3(a.H, R), dim3(256), 0, st, a);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int px_bonus_launch(cudaStream_t st, dim3 grid, const PxBonus& a) {
    launch_hi(px_bonus_kernel, grid, dim3(PT_THREADS), 0, st, a);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int px_value_launch(cudaStream_t st, int R, int H, double b, const double* sd, double* value) {
    launch_hi(px_value_kernel, dim3((R + 127) / 128), dim3(128), 0, st, R, H, b, sd, value);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}
