// particles_cscore.cu -- the whitening reverse of the score-function gradient over consistent function samples
// (pilco_particles_consistent_score_grad_rollout, DESIGN.md section 25).
// Per (particle row, output e) the consistent forward (fs_cond_kernel, particles.cu) leaves the packed rows l_ts (s < t)
// and the pivots piv_t = sqrt(d2_t) (0 for a degenerate column); with f_t and x held fixed the surrogate
//   J = (1/P) sum_p sum_{t<H-1, piv_t>0} w_pt (-eps_t(theta)^2 / 2 - log piv_t(theta)),
//   eps_t(theta) = (f_t - mean'_t(theta)) / piv_t(theta),  mean'_t = mu_t + sum_{s<t} l_ts eps_s
// moves the whitened residuals eps_s with theta.  Its reverse, t = H-2 .. 0, with eps_bar = 0 at the start:
//   piv_t > 0:  eps_bar_t -= w_t eps_t;  m_bar_t = -eps_bar_t / piv_t;  v_bar_t = (-w_t - eps_bar_t eps_t) / (2 d2_t);
//               eps_bar_s += m_bar_t l_ts for s < t
//   piv_t = 0:  m_bar_t = v_bar_t = 0 (tau rule: a deterministic step has no likelihood ratio)
// m_bar_t and v_bar_t are then the cotangents of step t's mean' and var' that fs_cond_bwd_kernel reads, with eps fixed
// inside it.  At the forward's point eps_t(theta) is the caller's eps_t, so only forward quantities are read.  v_bar_t is
// formed as (w_t (eps_t^2 - 1) - eps_bar'_t eps_t) / (2 d2_t), eps_bar'_t the later steps' share and d2_t the forward's
// var'_t: with no later share (H = 2) m_bar and v_bar are then bitwise ps_cot_kernel's at the same variance.
#include "particles.cuh"

#define PC_WARPS 8                      // warps (particle rows) per CTA, as fs_cond_kernel

// grid (ceil(P / PC_WARPS), E, R), one warp per (particle p of restart r = blockIdx.z, output e).  eps_bar_s lives in
// m_bar's slot of step s until step s is reached: lane s % 32 owns the slots s, s + 32, ..., so every slot is read
// and written by one thread only, and eps_bar_s is the sum over t = H-2 .. s+1 in that order.
__global__ void __launch_bounds__(PC_WARPS * 32) pc_white_kernel(PcWhite a) {
    PDL_ENTRY();
    const int lane = threadIdx.x & 31, p = blockIdx.x * PC_WARPS + (threadIdx.x >> 5), e = blockIdx.y, r = blockIdx.z;
    if (p >= a.P) return;
    const int H = a.H, Ds = a.Ds, Hm = H - 1;
    const size_t T = a.T, row = (size_t)r * a.P + p, EP = (size_t)Ds * T, pe = (size_t)e * T + row;
    const size_t TE = (size_t)T * Ds, o = row * Ds + e;                // step t's (row, e) at o + t TE
    double* mb = a.mbar + o;
    double* vb = a.vbar + o;
    const double* ep = a.eps + (size_t)p * H * Ds + e;                  // eps_t at ep[t Ds]
    for (int s = lane; s < Hm; s += 32) mb[(size_t)s * TE] = 0.0;
    for (int t = Hm - 1; t >= 0; --t) {
        const double* Lt = a.L + (size_t)t * (t + 1) / 2 * EP + pe;    // row t: entry s at Lt[s EP]
        const double piv = Lt[(size_t)t * EP];
        double m = 0.0;
        if (lane == (t & 31)) {
            double v = 0.0;
            if (piv > 0.0) {                                            // w_t as ps_cot_kernel forms it
                const double G = a.G[(size_t)t * T + row];
                const double w = a.P > 1 ? G - (a.S[(size_t)r * H + t] - G) / (a.P - 1) : G;
                const double et = ep[(size_t)t * Ds];
                const double later = mb[(size_t)t * TE], d2 = a.var[(size_t)t * TE + o];
                m = -fma(-w, et, later) / piv;
                v = fma(-later, et, w * (et * et - 1.0)) / (2.0 * d2);
            }
            mb[(size_t)t * TE] = m;
            vb[(size_t)t * TE] = v;
        }
        if (!(piv > 0.0)) continue;                                     // warp-uniform: nothing to pass on
        m = __shfl_sync(0xffffffffu, m, t & 31);
        for (int s = lane; s < t; s += 32) mb[(size_t)s * TE] = fma(m, Lt[(size_t)s * EP], mb[(size_t)s * TE]);
    }
}

int pc_white_launch(cudaStream_t st, int R, const PcWhite& a) {
    if (a.H < 2) return PILCO_OK;
    launch_hi(pc_white_kernel, dim3((a.P + PC_WARPS - 1) / PC_WARPS, a.Ds, R), dim3(PC_WARPS * 32), 0, st, a);
    CUDA_LAUNCH_CHECK();
    return PILCO_OK;
}
