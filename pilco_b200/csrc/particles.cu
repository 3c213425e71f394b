// particles.cu -- Monte Carlo particle rollout of the learnt dynamics under the policy (fp64):
//   pilco_particles_rollout   P particles x H steps of the Markov chain whose Gaussian marginals the moment-matching
//                             cascade (rollout.cu) approximates; the caller supplies x0 and the standard normals
//   u_t = squash(pi(x_t)),  x_{t+1} = x_t + mu(x~_t) + sqrt(max(var(x~_t), 0)) o eps_t,  x~_t = [x_t, u_t]
// Launch sequence (one stream, graph-capturable, no host sync; DESIGN.md section 11):
//   pt_step<0>, predict, pt_step<1>, predict, ..., predict, pt_step<H>
// pt_step_kernel is one thread per particle: it closes the previous step from the predict outputs, writes traj[:, t],
// and for t < H evaluates the reward terms at the point x_t, the policy and the predict input x~_t; at t = H it sums
// the return.  The O(n^2) work per step is pilco_gp_predict (predict.cu) at T = P.
#include "common.cuh"
#include "risk_math.cuh"

#define PT_THREADS 128
#define PT_MAX_P   (65535 * 32)         // pilco_gp_predict's T limit
#define PT_RBF_VAR 1e-6                 // output variance of the deterministic-GP policy (mode 1, mm_finish_device)
#define PT_INV_PI  0.31830988618379067154

struct PtDev {
    int P, H, Ds, U, t;
    int pol_kind, squash;
    const double* maxa;
    const double* W; const double* b;                   // linear policy [U,Ds], [U]
    const double* C; const double* ell; const double* sf2; const double* beta; int bf;   // RBF policy
    int n_rewards, n_mult; pilco_reward_term rewards[8]; double mult_mu;
    const double* x0; const double* eps;
    double* traj; double* act; double* step_reward; double* step_risk; double* ret;
    double* xt;                                         // predict input [P,D]
    const double* mean; const double* var;              // predict outputs [P,Ds]
};

// one reward term at the point x (registers; xg = the same point in global memory, for the box's indexed reads):
// the closed forms of small_kernels.cuh at s = 0
__device__ __forceinline__ double pt_reward_value(const pilco_reward_term& rt, const double (&x)[MAXD], const double* xg,
                                                  int Ds) {
    if (rt.kind == PILCO_REWARD_BOX) return risk_box_point(rt.W, xg);
    if (rt.kind == PILCO_REWARD_LINEAR) {
        double mu = 0.0;
#pragma unroll
        for (int i = 0; i < MAXD; ++i) if (i < Ds) mu = fma(x[i], rt.W[i], mu);
        return mu;
    }
    double v[MAXD];                                     // exp(-0.5 (x-t)' W (x-t)), dev_exp_reward's order
#pragma unroll
    for (int i = 0; i < MAXD; ++i) v[i] = i < Ds ? x[i] - rt.t[i] : 0.0;
    double quad = 0.0;
#pragma unroll
    for (int i = 0; i < MAXD; ++i) {
        if (i < Ds) {
            double wy = 0.0;
#pragma unroll
            for (int k = 0; k < MAXD; ++k) if (k < Ds) wy = fma(rt.W[i * Ds + k], v[k], wy);
            quad = fma(v[i], wy, quad);
        }
    }
    return exp(-0.5 * quad);
}

// grid ceil(P / 128), one thread per particle
__global__ void __launch_bounds__(PT_THREADS) pt_step_kernel(PtDev a) {
    PDL_ENTRY();
    const int p = blockIdx.x * PT_THREADS + threadIdx.x;
    if (p >= a.P) return;
    const int Ds = a.Ds, U = a.U, D = Ds + U, t = a.t, H = a.H;
    double* tr = a.traj + ((size_t)p * (H + 1) + t) * Ds;
    double x[MAXD];
    if (t == 0) {
#pragma unroll
        for (int d = 0; d < MAXD; ++d) x[d] = d < Ds ? a.x0[(size_t)p * Ds + d] : 0.0;
    } else {                                            // close step t-1
        const double* xp = tr - Ds;
        const double* mu = a.mean + (size_t)p * Ds;
        const double* var = a.var + (size_t)p * Ds;
        const double* ep = a.eps + ((size_t)p * H + (t - 1)) * Ds;
#pragma unroll
        for (int d = 0; d < MAXD; ++d) {
            if (d < Ds) {
                const double v = var[d];
                x[d] = fma(sqrt(v < 0.0 ? 0.0 : v), ep[d], xp[d] + mu[d]);      // NaN stays NaN
            } else x[d] = 0.0;
        }
    }
#pragma unroll
    for (int d = 0; d < MAXD; ++d) if (d < Ds) tr[d] = x[d];
    const size_t ph = (size_t)p * H;
    if (t == H) {                                       // return: step order, as ro_reward_sum_kernel
        double s = 0.0;
        for (int tt = 0; tt < H; ++tt) s += a.step_reward[ph + tt];
        if (a.n_mult > 0) {
            double mult = 1.0;
            for (int tt = 0; tt < H; ++tt) mult *= 1.0 - a.step_risk[ph + tt];
            s += a.mult_mu * (1.0 - mult);
        }
        a.ret[p] = s;
        return;
    }
    double rew = 0.0, risk = 0.0;                       // at the pre-step state (pilco.py:130-134)
    for (int k = 0; k < a.n_rewards; ++k) {
        const pilco_reward_term& rt = a.rewards[k];
        const double v = pt_reward_value(rt, x, tr, Ds);
        if (rt.channel == PILCO_CHANNEL_MULT) risk = fma(rt.coef, v, risk);
        else rew = fma(rt.coef, v, rew);
    }
    a.step_reward[ph + t] = rew;
    a.step_risk[ph + t] = risk;
    double* xo = a.xt + (size_t)p * D;
#pragma unroll
    for (int d = 0; d < MAXD; ++d) if (d < Ds) xo[d] = x[d];
    double* ao = a.act + (ph + t) * U;
    // squash_sin at a point with the policy's output variance su: maxa exp(-su/2) sin(u)  (dev_squash_sin's form).
    // sin(u) as sinpi(u / pi): its argument reduction is exact, so the kernel carries no Payne-Hanek slow path (whose
    // table lives in local memory); the rounding of u / pi moves the angle by |u| 1.1e-16 at most.
    const double su = a.pol_kind == PILCO_POLICY_RBF ? PT_RBF_VAR : 0.0;
    for (int j = 0; j < U; ++j) {
        double u;
        if (a.pol_kind == PILCO_POLICY_LINEAR) {        // dev_linear_action's order
            u = a.b[j];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) if (d < Ds) u = fma(a.W[j * Ds + d], x[d], u);
        } else {                                        // sum_i beta_ji sf2_j exp(-0.5 |(x - c_i) / ell_j|^2)
            double il[MAXD];
#pragma unroll
            for (int d = 0; d < MAXD; ++d) il[d] = d < Ds ? 1.0 / a.ell[j * Ds + d] : 0.0;
            const double sf2 = a.sf2[j];
            const double* be = a.beta + (size_t)j * a.bf;
            u = 0.0;
            for (int i = 0; i < a.bf; ++i) {
                const double* c = a.C + (size_t)i * Ds;
                double d2 = 0.0;
#pragma unroll
                for (int d = 0; d < MAXD; ++d) if (d < Ds) { const double q = (x[d] - c[d]) * il[d]; d2 = fma(q, q, d2); }
                u = fma(sf2 * exp(-0.5 * d2), be[i], u);
            }
        }
        if (a.squash) u = a.maxa[j] * exp(-0.5 * su) * sinpi(u * PT_INV_PI);
        ao[j] = u;
        xo[Ds + j] = u;
    }
}

struct PtWs { size_t xt, mean, var, pws, pws_bytes, total; };     // offsets in doubles; total and pws_bytes in bytes

static PtWs pt_ws_layout(const pilco_particles* pr) {
    const size_t P = pr->P, Ds = pr->pol.Ds, D = pr->dyn.D;
    PtWs L; size_t o = 0;
    auto take = [&](size_t len) { const size_t at = o; o += (len + 1) & ~(size_t)1; return at; };
    L.xt = take(P * D); L.mean = take(P * Ds); L.var = take(P * Ds);
    L.pws = o;
    L.pws_bytes = pilco_gp_predict_workspace_bytes(pr->dyn.n, pr->dyn.D, (int)Ds, pr->P, 0);
    L.total = o * sizeof(double) + L.pws_bytes;
    return L;
}

static bool pt_sizes_ok(const pilco_particles* pr) {
    return pr->P >= 1 && pr->P <= PT_MAX_P && pr->H >= 0 && pr->dyn.n >= 1 && pr->dyn.D >= 1 && pr->dyn.D <= MAXD &&
           pr->pol.Ds >= 1 && pr->pol.U >= 1 && pr->pol.Ds <= MAXE;
}

static int pt_check(const pilco_particles* pr) {
    if (!pr) return PILCO_ERR_NULL;
    if (pr->P < 1 || pr->P > PT_MAX_P || pr->H < 0) return PILCO_ERR_DIM;
    const pilco_gp_model& g = pr->dyn;
    if (!g.X || !g.ell || !g.sf2 || !g.beta) return PILCO_ERR_NULL;
    if (g.mode != 0 || !g.iK || g.X_bs || g.ell_bs || g.sf2_bs || g.beta_bs) return PILCO_ERR_UNSUPPORTED;
    if (g.n < 1 || g.D < 1 || g.D > MAXD || g.E < 1 || g.E > MAXE || g.ldk < pad64(g.n)) return PILCO_ERR_DIM;
    const pilco_policy& pol = pr->pol;
    const int Ds = pol.Ds, U = pol.U;
    if (Ds < 1 || U < 1 || Ds + U != g.D || g.E != Ds) return PILCO_ERR_DIM;
    if (pol.kind == PILCO_POLICY_LINEAR) {
        if (!pol.W || !pol.b) return PILCO_ERR_NULL;
        if (pol.W_bs || pol.b_bs) return PILCO_ERR_UNSUPPORTED;
    } else if (pol.kind == PILCO_POLICY_RBF) {
        const pilco_gp_model& r = pol.rbf;
        if (!r.X || !r.ell || !r.sf2 || !r.beta) return PILCO_ERR_NULL;
        if (r.mode != 1 || r.X_bs || r.ell_bs || r.sf2_bs || r.beta_bs) return PILCO_ERR_UNSUPPORTED;
        if (r.n < 1 || r.D != Ds || r.E != U) return PILCO_ERR_DIM;
    } else return PILCO_ERR_UNSUPPORTED;
    if (pol.squash && !pol.max_action) return PILCO_ERR_NULL;
    if (pr->n_rewards < 1 || pr->n_rewards > 8) return PILCO_ERR_DIM;
    for (int k = 0; k < pr->n_rewards; ++k) {
        const pilco_reward_term& rt = pr->rewards[k];
        if (!rt.W) return PILCO_ERR_NULL;
        if (rt.kind != PILCO_REWARD_EXP && rt.kind != PILCO_REWARD_LINEAR && rt.kind != PILCO_REWARD_BOX) return PILCO_ERR_UNSUPPORTED;
        if (rt.channel != PILCO_CHANNEL_ADD && rt.channel != PILCO_CHANNEL_MULT) return PILCO_ERR_UNSUPPORTED;
        if (rt.kind == PILCO_REWARD_EXP && !rt.t) return PILCO_ERR_NULL;
    }
    if (!pr->x0 || !pr->eps || !pr->traj || !pr->act || !pr->step_reward || !pr->step_risk || !pr->ret || !pr->ws)
        return PILCO_ERR_NULL;
    if (((uintptr_t)g.iK & 15) || (g.ldk & 1) || ((uintptr_t)pr->ws & 15)) return PILCO_ERR_ALIGN;   // predict's TMA rows
    const PtWs L = pt_ws_layout(pr);
    if (L.pws_bytes == 0) return PILCO_ERR_DIM;
    if (pr->ws_bytes < L.total) return PILCO_ERR_WORKSPACE;
    return PILCO_OK;
}

extern "C" {

size_t pilco_particles_workspace_bytes(const pilco_particles* pr) {
    if (!pr || !pt_sizes_ok(pr)) return 0;
    const PtWs L = pt_ws_layout(pr);
    return L.pws_bytes ? L.total : 0;
}

int pilco_particles_rollout(const pilco_particles* pr, pilco_stream_t stream) {
    const int rc0 = pt_check(pr);
    if (rc0) return rc0;
    const PtWs L = pt_ws_layout(pr);
    cudaStream_t st = (cudaStream_t)stream;
    double* ws = (double*)pr->ws;
    const pilco_policy& pol = pr->pol;
    PtDev a;
    a.P = pr->P; a.H = pr->H; a.Ds = pol.Ds; a.U = pol.U;
    a.pol_kind = pol.kind; a.squash = pol.squash; a.maxa = pol.max_action;
    a.W = pol.W; a.b = pol.b;
    a.C = pol.rbf.X; a.ell = pol.rbf.ell; a.sf2 = pol.rbf.sf2; a.beta = pol.rbf.beta; a.bf = pol.rbf.n;
    a.n_rewards = pr->n_rewards; a.n_mult = 0;
    for (int k = 0; k < 8; ++k) a.rewards[k] = pr->rewards[k];
    for (int k = 0; k < pr->n_rewards; ++k) a.n_mult += pr->rewards[k].channel == PILCO_CHANNEL_MULT;
    a.mult_mu = pr->mult_mu;
    a.x0 = pr->x0; a.eps = pr->eps;
    a.traj = pr->traj; a.act = pr->act; a.step_reward = pr->step_reward; a.step_risk = pr->step_risk; a.ret = pr->ret;
    a.xt = ws + L.xt; a.mean = ws + L.mean; a.var = ws + L.var;
    const dim3 grid((pr->P + PT_THREADS - 1) / PT_THREADS);
    for (int t = 0; t <= pr->H; ++t) {
        a.t = t;
        launch_hi(pt_step_kernel, grid, dim3(PT_THREADS), 0, st, a);
        CUDA_LAUNCH_CHECK();
        if (t == pr->H) break;
        const int rc = pilco_gp_predict(&pr->dyn, 0, pol.Ds, pr->P, ws + L.xt, ws + L.mean, ws + L.var, 0,
                                        ws + L.pws, L.pws_bytes, stream);
        if (rc) return rc;
    }
    return PILCO_OK;
}

}  // extern "C"
