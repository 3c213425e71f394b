// closed_forms.cu -- C-ABI entry points for the closed-form moment computations (batched over R):
// squash_sin (controllers.py:13-36), LinearController (controllers.py:46-58),
// ExponentialReward (rewards.py:19-51).
#include "small_kernels.cuh"

__global__ void __launch_bounds__(128) squash_kernel(int U, const double* m, const double* s, const double* maxa,
                                                     double* M, double* S, double* C) {
    const size_t r = blockIdx.x;
    dev_squash_sin(U, m + r * U, s + r * U * U, maxa, M + r * U, S + r * U * U, C + r * U * U);
}

__global__ void __launch_bounds__(128) linear_kernel(int Ds, int U, const double* W, long long W_bs,
                                                     const double* b, long long b_bs,
                                                     const double* m, const double* s,
                                                     double* M, double* S, double* V) {
    __shared__ SmallScratch sc;
    const size_t r = blockIdx.x;
    dev_linear_action(Ds, U, W + r * W_bs, b + r * b_bs, m + r * Ds, s + r * Ds * Ds,
                      M + r * U, S + r * U * U, V + r * Ds * U, sc);
}

__global__ void __launch_bounds__(128) exp_reward_kernel(int Ds, const double* W, const double* t,
                                                         const double* m, const double* s,
                                                         double* muR, double* sR) {
    __shared__ SmallScratch sc;
    const size_t r = blockIdx.x;
    const double mu = dev_exp_reward(Ds, W, t, m + r * Ds, s + r * Ds * Ds, sR ? sR + r : nullptr, sc);
    if (threadIdx.x == 0) muR[r] = mu;
}

__global__ void __launch_bounds__(32) box_risk_kernel(int Ds, const double* prm, const double* m, const double* s,
                                                      double* risk, double* dmo, double* dvo) {
    const size_t r = blockIdx.x;
    if (threadIdx.x != 0) return;
    double dm[RISK_MAX_DIMS], dv[RISK_MAX_DIMS];
    const bool grad = dmo != nullptr || dvo != nullptr;
    risk[r] = risk_box_eval(Ds, prm, m + r * Ds, s + r * Ds * Ds, grad ? dm : nullptr, grad ? dv : nullptr);
    if (grad) {
        for (int i = 0; i < Ds; ++i) { if (dmo) dmo[r * Ds + i] = 0.0; if (dvo) dvo[r * Ds + i] = 0.0; }
        const int nd = (int)prm[0];
        for (int k = 0; k < nd; ++k) {
            const int d = (int)prm[3 + 3 * k];
            if (dmo) dmo[r * Ds + d] += dm[k];
            if (dvo) dvo[r * Ds + d] += dv[k];
        }
    }
}

__global__ void __launch_bounds__(128) tg_moments_kernel(TrigMap tm, const double* m, const double* s,
                                                         double* M, double* S, double* C) {
    const size_t r = blockIdx.x, Ds = tm.Ds, Dh = trig_dh(tm);
    dev_trig(tm, m + r * Ds, s + r * Ds * Ds, M + r * Dh, S + r * Dh * Dh, C + r * Ds * Dh);
}

extern "C" {

int pilco_squash_sin(int U, int R, const double* m, const double* s, const double* max_action,
                     double* M, double* S, double* C, pilco_stream_t stream) {
    if (!m || !s || !max_action || !M || !S || !C) return PILCO_ERR_NULL;
    if (U < 1 || U > MAXD || R < 1) return PILCO_ERR_DIM;
    squash_kernel<<<R, 128, 0, (cudaStream_t)stream>>>(U, m, s, max_action, M, S, C);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int pilco_linear_action(int Ds, int U, int R, const double* W, long long W_bs, const double* b, long long b_bs,
                        const double* m, const double* s, double* M, double* S, double* V,
                        pilco_stream_t stream) {
    if (!W || !b || !m || !s || !M || !S || !V) return PILCO_ERR_NULL;
    if (Ds < 1 || Ds > MAXD || U < 1 || U > MAXD || R < 1) return PILCO_ERR_DIM;
    linear_kernel<<<R, 128, 0, (cudaStream_t)stream>>>(Ds, U, W, W_bs, b, b_bs, m, s, M, S, V);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int pilco_exp_reward(int Ds, int R, const double* W, const double* t, const double* m, const double* s,
                     double* muR, double* sR, int* info, pilco_stream_t stream) {
    (void)info;
    if (!W || !t || !m || !s || !muR) return PILCO_ERR_NULL;
    if (Ds < 1 || Ds > MAXD || R < 1) return PILCO_ERR_DIM;
    exp_reward_kernel<<<R, 128, 0, (cudaStream_t)stream>>>(Ds, W, t, m, s, muR, sR);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int pilco_box_risk(int Ds, int R, const double* prm, const double* m, const double* s,
                   double* risk, double* drisk_dm, double* drisk_dv, pilco_stream_t stream) {
    if (!prm || !m || !s || !risk) return PILCO_ERR_NULL;
    if (Ds < 1 || Ds > MAXD || R < 1) return PILCO_ERR_DIM;
    box_risk_kernel<<<R, 32, 0, (cudaStream_t)stream>>>(Ds, prm, m, s, risk, drisk_dm, drisk_dv);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

int pilco_trig_moments(int Ds, int R, const pilco_angles* ang, const double* m, const double* s,
                       double* M, double* S, double* C, pilco_stream_t stream) {
    if (!m || !s || !M || !S || !C) return PILCO_ERR_NULL;
    TrigMap tm;
    const int A = ang ? ang->A : 0;
    if (R < 1 || trig_map_make(Ds, A, ang ? ang->dims : nullptr, &tm) || Ds + A > MAXD) return PILCO_ERR_DIM;
    tg_moments_kernel<<<R, 128, 0, (cudaStream_t)stream>>>(tm, m, s, M, S, C);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}

}  // extern "C"
