// mm_forward.cu -- host side of pilco_mm_forward (C ABI) + shared launcher.
#include <stdlib.h>
#include <initializer_list>
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
    // 4 (default): 3 CTAs/SM, two row octets per warp on off-diagonal pairs as ONE 16-row tile on the 16x8 MMA shapes
    // (mm_tile_m16_kernel); 3: 3 CTAs/SM, two row octets per warp on DMMA.8x8x4 (80 registers); 1: 3 CTAs/SM, one octet per
    // warp (the round-1 kernel); 0: 2 CTAs/SM, two octets; 2: 4 CTAs/SM, one octet.  PILCO_TILE_VARIANT selects (tuning switch).
    static const int variant = [] {
        const char* e = getenv("PILCO_TILE_VARIANT");
        return e && e[0] >= '0' && e[0] <= '4' ? e[0] - '0' : 4;
    }();
    static const int rpc_env = [] { const char* e = getenv("PILCO_TILE_RPC"); return e ? atoi(e) : 0; }();   // 0: automatic
    if (pilco_smem_optin<mm_tile_kernel<KS, 2>, mm_tile_kernel<KS, 3>, mm_tile_kernel<KS, 4>, mm_tile_kernel<KS, 3, true>,
                         mm_tile_m16_kernel<KS>>((int)mm_tile_smem_bytes(TILE_CM, 20)))
        return PILCO_ERR_LAUNCH;
    const size_t smem = mm_tile_smem_bytes(p.L.np, p.L.ldz);
    int rpc = mm_tile_rpc(p.L.NB, p.L.P, p.R, pilco_sm_count());   // row blocks per CTA
    if (rpc_env > 0) rpc = rpc_env;
    if (rpc > p.L.NB) rpc = p.L.NB;
    dim3 grid((p.L.NB + rpc - 1) / rpc, p.L.P, p.R);
    // High priority only for a launch of at most half the SMs' worth of CTAs (the RBF policy's few pairs: glue on the step's
    // serial path).  A dynamics tile launch of a sub-batch (220 CTAs at the metric shape) is bulk work even though it fills
    // the machine less than twice: at high priority its queued CTAs would keep the setup and glue kernels of the other
    // sub-batches from the slots that free up, and their steps would stall behind it (DESIGN §6).
    const bool hi = (long long)grid.x * grid.y * grid.z <= pilco_sm_count() / 2;
    if (variant == 4) launch_pri(hi, mm_tile_m16_kernel<KS>, grid, dim3(256), smem, st, p, rpc);
    else if (variant == 3) launch_pri(hi, mm_tile_kernel<KS, 3, true>, grid, dim3(256), smem, st, p, rpc);
    else if (variant == 2) launch_pri(hi, mm_tile_kernel<KS, 4>, grid, dim3(256), smem, st, p, rpc);
    else if (variant == 1) launch_pri(hi, mm_tile_kernel<KS, 3>, grid, dim3(256), smem, st, p, rpc);
    else launch_pri(hi, mm_tile_kernel<KS, 2>, grid, dim3(256), smem, st, p, rpc);
    return PILCO_OK;
}

int mm_forward_launch(const MMParams& p, cudaStream_t st, bool with_finish, cudaEvent_t* ev) {
    if (ev) cudaEventRecord(ev[0], st);
    ks_dispatch(p.gp.D, [&](auto ks) { mm_setup_launch<4 * ks, false>(p, st); });
    CUDA_LAUNCH_CHECK();
    if (ev) cudaEventRecord(ev[1], st);
    const int rc = p.tape != nullptr ? mm_tape_tile_launch(p, st)      // taped forward: same sums + what the reverse sweep needs
                                     : ks_dispatch(p.gp.D, [&](auto ks) { return launch_tile<ks>(p, st); });
    if (rc) return rc;
    CUDA_LAUNCH_CHECK();
    if (ev) cudaEventRecord(ev[2], st);
    if (with_finish) {
        launch_hi(mm_finish_kernel, dim3(p.R), dim3(128), 0, st, p);
        CUDA_LAUNCH_CHECK();
    }
    if (ev) cudaEventRecord(ev[3], st);
    return PILCO_OK;
}

// Argument checks of the four forward entry points, in this order: the model, the pointers that must not be null, R,
// the taped path's shapes, workspace and tape sizes, then 16-byte alignment of both (the TMA bulk copies need it).
// tape: null for the untaped entry points.
static int mm_forward_check(const pilco_gp_model* gp, int R, std::initializer_list<const void*> required,
                            const void* ws, size_t ws_bytes, const void* tape, size_t tape_bytes) {
    const int rc = mm_check_model(gp);
    if (rc) return rc;
    for (const void* q : required)
        if (!q) return PILCO_ERR_NULL;
    if (R < 1) return PILCO_ERR_DIM;
    if (tape && !mm_tape_supported(gp->n, gp->D)) return PILCO_ERR_UNSUPPORTED;
    if (ws_bytes < pilco_mm_workspace_bytes(gp->n, gp->D, gp->E, R)) return PILCO_ERR_WORKSPACE;
    if (tape && tape_bytes < pilco_mm_tape_bytes(gp->n, gp->D, gp->E, R)) return PILCO_ERR_WORKSPACE;
    if ((((uintptr_t)ws) | ((uintptr_t)tape)) & 15) return PILCO_ERR_ALIGN;
    return PILCO_OK;
}

// Diagnostic: the launch sequence of pilco_mm_forward (or, with a tape, pilco_mm_forward_taped) with CUDA events around
// its three stages (ms_out[0..2] = setup, tile, finish).  Synchronises; never call it in a captured region.
static int mm_forward_profile(const MMParams& p, float* ms_out, cudaStream_t st) {
    cudaEvent_t ev[4];
    for (cudaEvent_t& e : ev) cudaEventCreate(&e);
    int rc = mm_forward_launch(p, st, true, ev);
    if (rc == PILCO_OK) {
        cudaEventSynchronize(ev[3]);
        for (int i = 0; i < 3; ++i) cudaEventElapsedTime(&ms_out[i], ev[i], ev[i + 1]);
    }
    for (cudaEvent_t& e : ev) cudaEventDestroy(e);
    if (rc == PILCO_OK && cudaGetLastError() != cudaSuccess) rc = PILCO_ERR_LAUNCH;
    return rc;
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
    const int rc = mm_forward_check(gp, R, {m, s, M, S, V, ws}, ws, ws_bytes, nullptr, 0);
    if (rc) return rc;
    return mm_forward_launch(mm_params(gp, R, m, gp->D, s, (long long)gp->D * gp->D, M, S, V, info, (double*)ws),
                             (cudaStream_t)stream, true);
}

int pilco_mm_forward_taped(const pilco_gp_model* gp, int R, const double* m, const double* s,
                           double* M, double* S, double* V, int* info,
                           void* ws, size_t ws_bytes, void* tape, size_t tape_bytes, pilco_stream_t stream) {
    const int rc = mm_forward_check(gp, R, {m, s, M, S, V, ws, tape}, ws, ws_bytes, tape, tape_bytes);
    if (rc) return rc;
    return mm_forward_launch(mm_params(gp, R, m, gp->D, s, (long long)gp->D * gp->D, M, S, V, info, (double*)ws,
                                       (double*)tape, mm_tape_layout(gp->n, gp->D, gp->E, R)),
                             (cudaStream_t)stream, true);
}

int pilco_mm_forward_profile(const pilco_gp_model* gp, int R, const double* m, const double* s,
                             double* M, double* S, double* V, int* info,
                             void* ws, size_t ws_bytes, float* ms_out, pilco_stream_t stream) {
    const int rc = mm_forward_check(gp, R, {m, s, M, S, V, ws, ms_out}, ws, ws_bytes, nullptr, 0);
    if (rc) return rc;
    return mm_forward_profile(mm_params(gp, R, m, gp->D, s, (long long)gp->D * gp->D, M, S, V, info, (double*)ws),
                              ms_out, (cudaStream_t)stream);
}

int pilco_mm_forward_taped_profile(const pilco_gp_model* gp, int R, const double* m, const double* s,
                                   double* M, double* S, double* V, int* info,
                                   void* ws, size_t ws_bytes, void* tape, size_t tape_bytes,
                                   float* ms_out, pilco_stream_t stream) {
    const int rc = mm_forward_check(gp, R, {m, s, M, S, V, ws, tape, ms_out}, ws, ws_bytes, tape, tape_bytes);
    if (rc) return rc;
    return mm_forward_profile(mm_params(gp, R, m, gp->D, s, (long long)gp->D * gp->D, M, S, V, info, (double*)ws,
                                        (double*)tape, mm_tape_layout(gp->n, gp->D, gp->E, R)),
                              ms_out, (cudaStream_t)stream);
}

}  // extern "C"

#ifdef PILCO_TILE_TIMING
extern "C" int pilco_debug_tile_timing(long long* host_out, int n) {
    return (int)cudaMemcpyFromSymbol(host_out, g_tile_timing, sizeof(long long) * (size_t)n);
}
#endif
