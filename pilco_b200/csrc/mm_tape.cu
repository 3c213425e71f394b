// mm_tape.cu -- host side of the taped moment match + the reverse sweep that consumes the tape.
// See mm_tape.cuh for the idea.  Reference: the policy gradient of pilco/models/pilco.py:47-50, 84-90 (TensorFlow
// autodiff through mgpr.py:91-149); numpy statement of exactly these formulas: oracle/staged.py:mm_backward_tape.
#include "mm_tape.cuh"

#include <stdlib.h>

template <int KS>
static int launch_tape_tile(const MMParams& p, cudaStream_t st) {
    // 4 (default): the 16x8-MMA kernel (mm_tape_tile_m16_kernel, <=128 regs); 0: the DMMA.8x8x4 kernel, <=128 regs; 1: <=96 regs,
    // 2 CTAs/SM; 2: <=80 regs, 2 CTAs/SM (padded smem); 3: <=80 regs, 3 CTAs/SM.  PILCO_TAPE_VARIANT selects (tuning switch).
    static const int variant = [] {
        const char* e = getenv("PILCO_TAPE_VARIANT");
        return e && e[0] >= '0' && e[0] <= '4' ? e[0] - '0' : 4;
    }();
    if (pilco_smem_optin<mm_tape_tile_m16_kernel<KS>, mm_tape_tile_kernel<KS, 256>, mm_tape_tile_kernel<KS, 304>,
                         mm_tape_tile_kernel<KS, 352>>(PILCO_MAX_SMEM_OPTIN))
        return PILCO_ERR_LAUNCH;
    size_t smem = mm_tape_smem_bytes(p.L.np, p.L.ldz);
    if (p.L.np > TAPE_MAX_NP || smem > PILCO_MAX_SMEM_OPTIN) return PILCO_ERR_UNSUPPORTED;
    const dim3 grid(p.TL.cs, p.L.P, p.R);
    const bool hi = pilco_small_grid(grid);
    if (variant == 4) launch_pri(hi, mm_tape_tile_m16_kernel<KS>, grid, dim3(256), smem, st, p);
    else if (variant == 0) launch_pri(hi, mm_tape_tile_kernel<KS, 256>, grid, dim3(256), smem, st, p);
    else if (variant == 1) launch_pri(hi, mm_tape_tile_kernel<KS, 304>, grid, dim3(256), smem, st, p);
    else {
        if (variant == 2 && smem < 80 * 1024) smem = 80 * 1024;    // 2 CTAs per SM
        launch_pri(hi, mm_tape_tile_kernel<KS, 352>, grid, dim3(256), smem, st, p);
    }
    return PILCO_OK;
}

int mm_tape_tile_launch(const MMParams& p, cudaStream_t st) {
    return ks_dispatch(p.gp.D, [&](auto ks) { return launch_tape_tile<ks>(p, st); });
}

template <int DP>
__global__ void __launch_bounds__(TB_THREADS, 3) mm_tape_bfinish_kernel(MMTapeBwd bp) {
    PDL_ENTRY();
    extern __shared__ __align__(16) double tb_dyn[];
    mm_tape_bfinish_task<DP>(bp, blockIdx.y, blockIdx.x, tb_dyn);
}

// sum the task partials -> gm, gs
__global__ void __launch_bounds__(128) mm_tape_breduce_kernel(MMTapeBwd bp) {
    PDL_ENTRY();
    const int r = blockIdx.x;
    mm_tape_reduce_device(bp.part + (size_t)r * mm_tape_bwd_part_doubles(bp.gp.D, bp.gp.E), bp.gp.E + bp.TL.P, bp.gp.D,
                          bp.gm + (size_t)r * bp.gm_rs, bp.gs + (size_t)r * bp.gs_rs, bp.accumulate);
}

int mm_tape_backward_launch(const MMTapeBwd& bp, cudaStream_t st, bool with_reduce) {
    const int E = bp.gp.E, R = bp.R;
    dim3 gf(E + bp.TL.P, R);
    const size_t smem = mm_tape_bfinish_smem_bytes(bp.TL.np, bp.gp.D);
    // large n: static + dynamic shared memory > 48 KB
    if (pilco_smem_optin<mm_tape_bfinish_kernel<4>, mm_tape_bfinish_kernel<8>, mm_tape_bfinish_kernel<12>,
                         mm_tape_bfinish_kernel<16>>(196 * 1024))
        return PILCO_ERR_LAUNCH;
    ks_dispatch(bp.gp.D, [&](auto ks) { launch_hi(mm_tape_bfinish_kernel<4 * ks>, gf, dim3(TB_THREADS), smem, st, bp); });
    CUDA_LAUNCH_CHECK();
    if (with_reduce) {
        launch_hi(mm_tape_breduce_kernel, dim3(R), dim3(128), 0, st, bp);
        CUDA_LAUNCH_CHECK();
    }
    return PILCO_OK;
}

extern "C" {

size_t pilco_mm_tape_bytes(int n, int D, int E, int R) {
    if (n < 1 || D < 1 || D > MAXD || E < 1 || E > MAXE || R < 1 || !mm_tape_supported(n, D)) return 0;
    return mm_tape_layout(n, D, E, R).per_r * (size_t)R * sizeof(double);
}

size_t pilco_mm_tape_bwd_workspace_bytes(int D, int E, int R) {
    if (D < 1 || D > MAXD || E < 1 || E > MAXE || R < 1) return 0;
    return mm_tape_bwd_part_doubles(D, E) * (size_t)R * sizeof(double);
}

int pilco_mm_backward_taped(const pilco_gp_model* gp, int R, const double* m, const double* s, const double* M,
                            const double* gM, const double* gS, const double* gV,
                            const void* tape, size_t tape_bytes, double* gm, double* gs,
                            void* ws, size_t ws_bytes, pilco_stream_t stream) {
    int rc = mm_check_model(gp);
    if (rc) return rc;
    if (!m || !s || !M || !gM || !gS || !gV || !tape || !gm || !gs || !ws) return PILCO_ERR_NULL;
    if (R < 1) return PILCO_ERR_DIM;
    if (!mm_tape_supported(gp->n, gp->D)) return PILCO_ERR_UNSUPPORTED;
    if (tape_bytes < pilco_mm_tape_bytes(gp->n, gp->D, gp->E, R)) return PILCO_ERR_WORKSPACE;
    if (ws_bytes < pilco_mm_tape_bwd_workspace_bytes(gp->D, gp->E, R)) return PILCO_ERR_WORKSPACE;
    if ((((uintptr_t)ws) | ((uintptr_t)tape)) & 15) return PILCO_ERR_ALIGN;
    const int D = gp->D;
    const MMTapeBwd bp = mm_tape_bwd_params(gp, R, m, D, s, (long long)D * D, M, gM, gS, gV, (const double*)tape,
                                            mm_tape_layout(gp->n, D, gp->E, R), (double*)ws, gm, D, gs, (long long)D * D);
    return mm_tape_backward_launch(bp, (cudaStream_t)stream, true);
}

}  // extern "C"
