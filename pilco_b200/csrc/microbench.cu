// microbench.cu -- fp64 pipe diagnostics used to set the roofline denominators:
//   which=0: DFMA only, 1: DMMA (m8n8k4) only, 2: DFMA+DMMA interleaved 1:1 (per-warp instruction counts),
//   3: exp_tab only, 4: libdevice exp only, 5: DMMA m16n8k8 only, 6: DMMA m16n8k16 only (Hopper's native fp64 MMA shapes:
//   what the fp64 tensor cores reach, against which the m8n8k4 rate of the tile kernels is compared), 7: DMMA m16n8k4 only,
//   8: DFMA+DMMA m16n8k16 interleaved 1:1, 9: DFMA+DMMA m16n8k8 interleaved 1:1 (does the 16x8 tensor path block DFMA issue
//   the way the 8x8x4 one does?).
// Returns achieved warp-instructions/s through *rate (DFMA or DMMA or exp evaluations per second, chip-wide).
#include "common.cuh"

// (dmma1684 / dmma1688 / dmma16816: common.cuh)

template <int WHICH>
__global__ void __launch_bounds__(256) fp64_pipe_kernel(int iters, double* sink) {
    __shared__ double tab[EXP_TAB_DOUBLES];
    exp_table_init(tab);
    __syncthreads();
    const double* ltab = EXP_LANE_TAB(tab, threadIdx.x);
    const double seed = 1.0 + 1e-9 * threadIdx.x;
    double a0 = seed, a1 = seed * 1.1, a2 = seed * 1.2, a3 = seed * 1.3, a4 = seed * 1.4, a5 = seed * 1.5, a6 = seed * 1.6, a7 = seed * 1.7;
    double c0 = 0, c1 = 0, c2 = 0, c3 = 0, c4 = 0, c5 = 0, c6 = 0, c7 = 0;
    const double m = 0.999999, b = 1e-7;
    for (int it = 0; it < iters; ++it) {
        if (WHICH == 0 || WHICH == 2 || WHICH == 8 || WHICH == 9) {
            a0 = fma(a0, m, b); a1 = fma(a1, m, b); a2 = fma(a2, m, b); a3 = fma(a3, m, b);
            a4 = fma(a4, m, b); a5 = fma(a5, m, b); a6 = fma(a6, m, b); a7 = fma(a7, m, b);
        }
        if (WHICH == 1 || WHICH == 2) {
            // distinct A/B registers per instruction (identical operands hit an operand-reuse fast path
            // and overstate the rate)
            dmma884(c0, c1, a0, a1); dmma884(c2, c3, a2, a3); dmma884(c4, c5, a4, a5); dmma884(c6, c7, a6, a7);
            dmma884(c0, c1, a1, a2); dmma884(c2, c3, a3, a4); dmma884(c4, c5, a5, a6); dmma884(c6, c7, a7, a0);
            if (WHICH == 1) { a0 += c1 * 1e-300; a3 += c2 * 1e-300; }
        }
        if (WHICH == 5 || WHICH == 6 || WHICH == 7 || WHICH == 8 || WHICH == 9) {
            // 8 MMAs per iteration into 4 independent accumulators, operands rotated (no identical-operand fast path)
            double x[8] = {a0, a1, a2, a3, a4, a5, a6, a7};
            double acc[4][4] = {{c0, c1, c2, c3}, {c4, c5, c6, c7}, {c1, c2, c3, c4}, {c5, c6, c7, c0}};
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (WHICH == 7) {
                    dmma1684(acc[k & 3], x[k & 7], x[(k + 1) & 7], x[(k + 4) & 7]);
                } else if (WHICH == 5 || WHICH == 9) {
                    const double av[4] = {x[k & 7], x[(k + 1) & 7], x[(k + 2) & 7], x[(k + 3) & 7]};
                    dmma1688(acc[k & 3], av, x[(k + 4) & 7], x[(k + 5) & 7]);
                } else {
                    const double av[8] = {x[k & 7], x[(k + 1) & 7], x[(k + 2) & 7], x[(k + 3) & 7],
                                          x[(k + 4) & 7], x[(k + 5) & 7], x[(k + 6) & 7], x[(k + 7) & 7]};
                    const double bv[4] = {x[(k + 3) & 7], x[(k + 5) & 7], x[(k + 6) & 7], x[(k + 1) & 7]};
                    dmma16816(acc[k & 3], av, bv);
                }
            }
            c0 = acc[0][0]; c1 = acc[0][1]; c2 = acc[0][2]; c3 = acc[0][3];
            c4 = acc[1][0] + acc[2][0]; c5 = acc[1][1] + acc[2][1]; c6 = acc[1][2] + acc[3][2]; c7 = acc[1][3] + acc[3][3];
            a0 += c1 * 1e-300; a3 += c2 * 1e-300;
        }
        if (WHICH == 3) {
            a0 = exp_scaled(a0 - 300.0, ltab); a1 = exp_scaled(a1 - 311.1, ltab); a2 = exp_scaled(a2 - 322.2, ltab); a3 = exp_scaled(a3 - 333.3, ltab);
            a4 = exp_scaled(a4 - 344.4, ltab); a5 = exp_scaled(a5 - 355.5, ltab); a6 = exp_scaled(a6 - 366.6, ltab); a7 = exp_scaled(a7 - 377.7, ltab);
        }
        if (WHICH == 4) {
            a0 = exp(a0 - 1.0); a1 = exp(a1 - 1.1); a2 = exp(a2 - 1.2); a3 = exp(a3 - 1.3);
            a4 = exp(a4 - 1.4); a5 = exp(a5 - 1.5); a6 = exp(a6 - 1.6); a7 = exp(a7 - 1.7);
        }
    }
    const double r = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7 + c0 + c1 + c2 + c3 + c4 + c5 + c6 + c7;
    if (r == 123.456) sink[0] = r;
}

extern "C" int pilco_microbench_fp64(int which, int iters, int blocks, double* sink_dev, float* ms_out, pilco_stream_t stream) {
    cudaStream_t st = (cudaStream_t)stream;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int rep = 0; rep < 2; ++rep) {
        cudaEventRecord(e0, st);
        switch (which) {
            case 0: fp64_pipe_kernel<0><<<blocks, 256, 0, st>>>(iters, sink_dev); break;
            case 1: fp64_pipe_kernel<1><<<blocks, 256, 0, st>>>(iters, sink_dev); break;
            case 2: fp64_pipe_kernel<2><<<blocks, 256, 0, st>>>(iters, sink_dev); break;
            case 3: fp64_pipe_kernel<3><<<blocks, 256, 0, st>>>(iters, sink_dev); break;
            case 5: fp64_pipe_kernel<5><<<blocks, 256, 0, st>>>(iters, sink_dev); break;
            case 6: fp64_pipe_kernel<6><<<blocks, 256, 0, st>>>(iters, sink_dev); break;
            case 7: fp64_pipe_kernel<7><<<blocks, 256, 0, st>>>(iters, sink_dev); break;
            case 8: fp64_pipe_kernel<8><<<blocks, 256, 0, st>>>(iters, sink_dev); break;
            case 9: fp64_pipe_kernel<9><<<blocks, 256, 0, st>>>(iters, sink_dev); break;
            default: fp64_pipe_kernel<4><<<blocks, 256, 0, st>>>(iters, sink_dev); break;
        }
        cudaEventRecord(e1, st);
        cudaEventSynchronize(e1);
    }
    if (cudaGetLastError() != cudaSuccess) return PILCO_ERR_LAUNCH;
    cudaEventElapsedTime(ms_out, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return PILCO_OK;
}
