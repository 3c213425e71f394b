// mm_forward.cu -- host side of pilco_mm_forward (C ABI) + shared launcher.
#include <stdlib.h>
#include "mm_tape.cuh"

int mm_check_model(const pilco_gp_model* gp) {
    if (!gp || !gp->X || !gp->ell || !gp->sf2 || !gp->beta) return PILCO_ERR_NULL;
    if (gp->n < 1 || gp->D < 1 || gp->D > MAXD || gp->E < 1 || gp->E > MAXE) return PILCO_ERR_DIM;
    if (gp->mode != 0 && gp->mode != 1) return PILCO_ERR_DIM;
    if (gp->mode == 0 && gp->iK) {
        if (gp->ldk < pad64(gp->n) || (gp->ldk & 1)) return PILCO_ERR_DIM;
        if (((uintptr_t)gp->iK) & 15) return PILCO_ERR_ALIGN;
    }
    return PILCO_OK;
}

template <int KS>
static int launch_tile(const MMParams& p, cudaStream_t st) {
    static bool configured_dev[PILCO_MAX_DEVICES] = {false};      // function attributes are per device
    // 4 (default): 3 CTAs/SM, two row octets per warp on off-diagonal pairs as ONE 16-row tile on the 16x8 MMA shapes
    // (mm_tile_m16_kernel); 3: 3 CTAs/SM, two row octets per warp on DMMA.8x8x4 (80 registers); 1: 3 CTAs/SM, one octet per
    // warp (the round-1 kernel); 0: 2 CTAs/SM, two octets; 2: 4 CTAs/SM, one octet.  PILCO_TILE_VARIANT selects (tuning switch).
    static int variant = 4;
    static int rpc_env = 0;          // 0: automatic
    bool& configured = configured_dev[pilco_current_device()];
    if (!configured) {
        const char* e = getenv("PILCO_TILE_VARIANT");       // tuning switches
        if (e && e[0] >= '0' && e[0] <= '4') variant = e[0] - '0';
        const char* e2 = getenv("PILCO_TILE_RPC");
        if (e2) rpc_env = atoi(e2);
        const int big = (int)mm_tile_smem_bytes(TILE_CM, 20);
        if (cudaFuncSetAttribute(mm_tile_kernel<KS, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, big) != cudaSuccess) return PILCO_ERR_LAUNCH;
        if (cudaFuncSetAttribute(mm_tile_kernel<KS, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, big) != cudaSuccess) return PILCO_ERR_LAUNCH;
        if (cudaFuncSetAttribute(mm_tile_kernel<KS, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, big) != cudaSuccess) return PILCO_ERR_LAUNCH;
        if (cudaFuncSetAttribute(mm_tile_kernel<KS, 3, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, big) != cudaSuccess) return PILCO_ERR_LAUNCH;
        if (cudaFuncSetAttribute(mm_tile_m16_kernel<KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, big) != cudaSuccess) return PILCO_ERR_LAUNCH;
        configured = true;
    }
    int rc = exp_table_upload();
    if (rc) return rc;
    const size_t smem = mm_tile_smem_bytes(p.L.np, p.L.ldz);
    // row blocks per CTA: a CTA's fixed cost (TMA staging of the columns and the exp table, barrier, first-load
    // latency: ~5 k cycles against ~16 k per 64-row sweep at the metric shape) is paid once for all its row blocks.
    // All of a pair's row blocks go to one CTA as soon as pairs x restarts still give every SM a CTA; smaller
    // launches keep enough CTAs to fill the machine (2 CTAs per SM).
    int rpc = p.L.NB;
    const long long pr = (long long)p.L.P * p.R, nsm = pilco_sm_count();
    if (pr < nsm) { rpc = (int)(((long long)p.L.NB * pr) / (2 * nsm)); if (rpc < 1) rpc = 1; }
    if (rpc_env > 0) rpc = rpc_env;
    if (rpc > p.L.NB) rpc = p.L.NB;
    dim3 grid((p.L.NB + rpc - 1) / rpc, p.L.P, p.R);
    const bool hi = pilco_small_grid(grid);          // e.g. the RBF policy's 3 pairs: glue, not bulk work
    if (variant == 4) launch_pri(hi, mm_tile_m16_kernel<KS>, grid, dim3(256), smem, st, p, rpc);
    else if (variant == 3) launch_pri(hi, mm_tile_kernel<KS, 3, true>, grid, dim3(256), smem, st, p, rpc);
    else if (variant == 2) launch_pri(hi, mm_tile_kernel<KS, 4>, grid, dim3(256), smem, st, p, rpc);
    else if (variant == 1) launch_pri(hi, mm_tile_kernel<KS, 3>, grid, dim3(256), smem, st, p, rpc);
    else launch_pri(hi, mm_tile_kernel<KS, 2>, grid, dim3(256), smem, st, p, rpc);
    return PILCO_OK;
}

int mm_forward_launch(const MMParams& p, cudaStream_t st, bool with_finish) {
    const int E = p.gp.E, D = p.gp.D;
    const int ks = ksteps_of(D);
    switch (ks) {
        case 1: mm_setup_launch<4, false>(p, st); break;
        case 2: mm_setup_launch<8, false>(p, st); break;
        case 3: mm_setup_launch<12, false>(p, st); break;
        default: mm_setup_launch<16, false>(p, st); break;
    }
    CUDA_LAUNCH_CHECK();
    int rc;
    if (p.tape != nullptr) rc = mm_tape_tile_launch(p, st);      // taped forward: same sums + what the reverse sweep needs
    else switch (ks) {
        case 1: rc = launch_tile<1>(p, st); break;
        case 2: rc = launch_tile<2>(p, st); break;
        case 3: rc = launch_tile<3>(p, st); break;
        default: rc = launch_tile<4>(p, st); break;
    }
    if (rc) return rc;
    CUDA_LAUNCH_CHECK();
    if (with_finish) {
        launch_hi(mm_finish_kernel, dim3(p.R), dim3(128), 0, st, p);
        CUDA_LAUNCH_CHECK();
    }
    return PILCO_OK;
}

extern "C" {

int pilco_pad_n(int n) { return pad64(n); }

size_t pilco_mm_workspace_bytes(int n, int D, int E, int R) {
    if (n < 1 || D < 1 || D > MAXD || E < 1 || E > MAXE || R < 1) return 0;
    const MMWs L = mm_ws_layout(n, D, E);
    return L.per_r * (size_t)R * sizeof(double);
}

int pilco_mm_forward(const pilco_gp_model* gp, int R, const double* m, const double* s,
                     double* M, double* S, double* V, int* info,
                     void* ws, size_t ws_bytes, pilco_stream_t stream) {
    int rc = mm_check_model(gp);
    if (rc) return rc;
    if (!m || !s || !M || !S || !V || !ws) return PILCO_ERR_NULL;
    if (R < 1) return PILCO_ERR_DIM;
    if (ws_bytes < pilco_mm_workspace_bytes(gp->n, gp->D, gp->E, R)) return PILCO_ERR_WORKSPACE;
    if (((uintptr_t)ws) & 15) return PILCO_ERR_ALIGN;
    MMParams p;
    p.gp = *gp; p.R = R; p.m = m; p.s = s; p.m_rs = gp->D; p.s_rs = (long long)gp->D * gp->D; p.M = M; p.S = S; p.V = V; p.info = info;
    p.ws = (double*)ws; p.L = mm_ws_layout(gp->n, gp->D, gp->E); p.bwd = 0; p.oQ = p.oC = p.oLd = 0;
    return mm_forward_launch(p, (cudaStream_t)stream, true);
}

// Diagnostic: same work as pilco_mm_forward (or, with a tape, pilco_mm_forward_taped), with CUDA events around the
// three launches (ms_out[0..2] = setup, tile, finish).  Synchronises; never call it in a captured region.
static int mm_forward_profile(MMParams& p, float* ms_out, cudaStream_t st) {
    cudaEvent_t ev[4];
    for (int i = 0; i < 4; ++i) cudaEventCreate(&ev[i]);
    const int ks = ksteps_of(p.gp.D);
    int rc;
    cudaEventRecord(ev[0], st);
    switch (ks) {
        case 1: mm_setup_launch<4, false>(p, st); break;
        case 2: mm_setup_launch<8, false>(p, st); break;
        case 3: mm_setup_launch<12, false>(p, st); break;
        default: mm_setup_launch<16, false>(p, st); break;
    }
    cudaEventRecord(ev[1], st);
    if (p.tape != nullptr) rc = mm_tape_tile_launch(p, st);
    else switch (ks) {
        case 1: rc = launch_tile<1>(p, st); break;
        case 2: rc = launch_tile<2>(p, st); break;
        case 3: rc = launch_tile<3>(p, st); break;
        default: rc = launch_tile<4>(p, st); break;
    }
    cudaEventRecord(ev[2], st);
    launch_hi(mm_finish_kernel, dim3(p.R), dim3(128), 0, st, p);
    cudaEventRecord(ev[3], st);
    cudaEventSynchronize(ev[3]);
    for (int i = 0; i < 3; ++i) cudaEventElapsedTime(&ms_out[i], ev[i], ev[i + 1]);
    for (int i = 0; i < 4; ++i) cudaEventDestroy(ev[i]);
    if (rc) return rc;
    if (cudaGetLastError() != cudaSuccess) return PILCO_ERR_LAUNCH;
    return PILCO_OK;
}

int pilco_mm_forward_profile(const pilco_gp_model* gp, int R, const double* m, const double* s,
                             double* M, double* S, double* V, int* info,
                             void* ws, size_t ws_bytes, float* ms_out, pilco_stream_t stream) {
    int rc = mm_check_model(gp);
    if (rc) return rc;
    if (!m || !s || !M || !S || !V || !ws || !ms_out) return PILCO_ERR_NULL;
    if (ws_bytes < pilco_mm_workspace_bytes(gp->n, gp->D, gp->E, R)) return PILCO_ERR_WORKSPACE;
    MMParams p;
    p.gp = *gp; p.R = R; p.m = m; p.s = s; p.m_rs = gp->D; p.s_rs = (long long)gp->D * gp->D;
    p.M = M; p.S = S; p.V = V; p.info = info;
    p.ws = (double*)ws; p.L = mm_ws_layout(gp->n, gp->D, gp->E); p.bwd = 0; p.oQ = p.oC = p.oLd = 0;
    return mm_forward_profile(p, ms_out, (cudaStream_t)stream);
}

int pilco_mm_forward_taped_profile(const pilco_gp_model* gp, int R, const double* m, const double* s,
                                   double* M, double* S, double* V, int* info,
                                   void* ws, size_t ws_bytes, void* tape, size_t tape_bytes,
                                   float* ms_out, pilco_stream_t stream) {
    int rc = mm_check_model(gp);
    if (rc) return rc;
    if (!m || !s || !M || !S || !V || !ws || !tape || !ms_out) return PILCO_ERR_NULL;
    if (!mm_tape_supported(gp->n, gp->D)) return PILCO_ERR_UNSUPPORTED;
    if (ws_bytes < pilco_mm_workspace_bytes(gp->n, gp->D, gp->E, R)) return PILCO_ERR_WORKSPACE;
    const MMTapeL TL = mm_tape_layout(gp->n, gp->D, gp->E, R);
    if (tape_bytes < TL.per_r * (size_t)R * sizeof(double)) return PILCO_ERR_WORKSPACE;
    MMParams p;
    p.gp = *gp; p.R = R; p.m = m; p.s = s; p.m_rs = gp->D; p.s_rs = (long long)gp->D * gp->D;
    p.M = M; p.S = S; p.V = V; p.info = info;
    p.ws = (double*)ws; p.L = mm_ws_layout(gp->n, gp->D, gp->E); p.bwd = 0; p.oQ = p.oC = p.oLd = 0;
    p.tape = (double*)tape; p.TL = TL;
    return mm_forward_profile(p, ms_out, (cudaStream_t)stream);
}

}  // extern "C"

#ifdef PILCO_TILE_TIMING
extern "C" int pilco_debug_tile_timing(long long* host_out, int n) {
    return (int)cudaMemcpyFromSymbol(host_out, g_tile_timing, sizeof(long long) * (size_t)n);
}
#endif
