// Host build of the tabularised Stokes drift of csrc/od_stokes.cuh for the CPU tests (tests/stokestab_host.py): the same
// per-element function the device kernel runs, one loop per launch.  Compiled with -ffp-contract=off, as the device build rounds
// every operation on its own.
#include <stdint.h>
#include <string.h>
#include "../../opendrift_b200/csrc/od_stokes.cuh"

using namespace od;

extern "C" {

int hs3_stokes_parameterised(int64_t n, const float* xwind, const float* ywind, const double* wf, int32_t n_wf, const double* hsc,
                             int32_t n_hs, float* us, float* vs, float* hs) {
    if (n < 0 || (!us) != (!vs) || (!us && !hs)) return -2;
    if ((us && (n_wf < 1 || n_wf > OD_TAB_MAX_COEF)) || (hs && (n_hs < 1 || n_hs > OD_TAB_MAX_COEF))) return -2;
    StokesTabParams p;
    memset(&p, 0, sizeof(p));
    p.n = n; p.xwind = xwind; p.ywind = ywind; p.us = us; p.vs = vs; p.hs = hs;
    if (us) { p.n_wf = n_wf; memcpy(p.wf, wf, sizeof(double) * n_wf); }
    if (hs) { p.n_hs = n_hs; memcpy(p.hsc, hsc, sizeof(double) * n_hs); }
    for (int64_t i = 0; i < n; ++i) stokes_tab_one(p, i);
    return 0;
}

}
