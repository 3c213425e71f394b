// Host build of pilco_b200/csrc/trig_math.cuh (the scalar formulas the device kernels execute for angular state
// dimensions) and the layout of pilco_angles, so that the CPU test suite can check both without a GPU.
// Test infrastructure only.
#include <stddef.h>
#include "../../include/pilco_b200.h"
#include "../../pilco_b200/csrc/trig_math.cuh"

extern "C" int trig_moments_host(int Ds, int A, const int* dims, const double* m, const double* s,
                                 double* M, double* S, double* C) {
    TrigMap tm;
    if (trig_map_make(Ds, A, dims, &tm)) return 1;
    const int Dh = trig_dh(tm);
    for (int k = 0; k < Dh; ++k) M[k] = trig_M_entry(tm, m, s, k);
    for (int e = 0; e < Dh * Dh; ++e) S[e] = trig_S_entry(tm, m, s, e / Dh, e % Dh);
    for (int e = 0; e < Ds * Dh; ++e) C[e] = trig_C_entry(tm, m, s, e / Dh, e % Dh);
    return 0;
}

extern "C" int trig_vjp_host(int Ds, int A, const int* dims, const double* m, const double* s, const double* gM,
                             const double* gS, const double* gC, double* gm, double* gs) {
    TrigMap tm;
    if (trig_map_make(Ds, A, dims, &tm)) return 1;
    for (int i = 0; i < Ds; ++i) gm[i] = trig_vjp_m(tm, m, s, gM, gS, gC, i);
    for (int e = 0; e < Ds * Ds; ++e) gs[e] = trig_vjp_s(tm, m, s, gM, gS, gC, e / Ds, e % Ds);
    return 0;
}

extern "C" void angles_layout(size_t* out) {
    out[0] = sizeof(pilco_angles);
    out[1] = offsetof(pilco_angles, A);
    out[2] = offsetof(pilco_angles, dims);
}
