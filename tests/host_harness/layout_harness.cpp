// Host build of the workspace-layout functions (pilco_b200/csrc/{mm_kernels,mm_backward,rollout}.cuh) so the CPU suite
// can check their invariants (ordering, alignment, sizes) against the sizes the shared library reports, and of the launch
// decisions of the moment match (tests/mm_cases.py states from them which kernel branch a case runs).
#include "../../pilco_b200/csrc/mm_backward.cuh"
#include "../../pilco_b200/csrc/rollout.cuh"

extern "C" {
// fills out[0..10): zeta, betap, Bq, Tpart, Wm, Wc, Qab, Ufrag, Arow, per_r (doubles); returns np
int layout_mm(int n, int D, int E, int ordered, unsigned long long* out) {
    const MMWs L = mm_ws_layout(n, D, E, ordered != 0);
    const size_t v[10] = {L.zeta, L.betap, L.Bq, L.Tpart, L.Wm, L.Wc, L.Qab, L.Ufrag, L.Arow, L.per_r};
    for (int i = 0; i < 10; ++i) out[i] = v[i];
    return L.np;
}
unsigned long long layout_bwd_per_r(int n, int D, int E, int need_param) { return mm_bws_layout(n, D, E, need_param).per_r; }
int layout_pair(int q, int* a, int* b) { int aa, bb; pair_decode(q, aa, bb); *a = aa; *b = bb; return pair_index(aa, bb); }
int layout_misc(int D, int* ldz, int* ks) { *ldz = ldz_of(D); *ks = ksteps_of(D); return pad64(D); }
// the launch decisions on a machine of nsm SMs: row blocks per forward tile CTA, row splits of the taped tile kernel,
// one fused setup launch or the two-stage form
int launch_tile_rpc(int NB, int P, int R, int nsm) { return mm_tile_rpc(NB, P, R, nsm); }
int launch_tape_splits(int n, int P, int R, int nsm) { return mm_tape_splits_on(n, P, R, nsm); }
int launch_setup_fused(int ntask, int R, int nsm) { return mm_setup_is_fused(ntask, R, nsm) ? 1 : 0; }
}
