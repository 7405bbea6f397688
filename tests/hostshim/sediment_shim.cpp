// Host build of SedimentDrift's device code for the CPU tests (tests/sediment_host.py): the settling variant of the mixing loop
// (mix_particle<PROJ, true> of csrc/od_mix.cuh) and resuspend_one, one loop per launch.  The mixing launch is hostshim.cpp's own
// (the same od_mix_args -> MixParams fill as od_kernels.cu), compiled into this library with its per-element call routed through
// settle_dispatch, which takes the settling variant while hs4_mix_settle runs.  Compiled with -ffp-contract=off, as the device
// build rounds every operation on its own.
#include <stdint.h>
#include "../../opendrift_b200/csrc/od_mix.cuh"

static const od::SettleParams* g_settle = nullptr;

template <bool PROJ = false>
static inline void settle_dispatch(const od::MixParams& p, int64_t i, const double* xs, const double* xy) {
    if (g_settle) od::mix_particle<PROJ, true>(p, i, xs, xy, g_settle);
    else od::mix_particle<PROJ>(p, i, xs, xy);
}

#define mix_particle settle_dispatch
#include "hostshim.cpp"
#undef mix_particle

extern "C" {

int hs4_mix_settle(const od_mix_args* a, const hs_group* g, const hs_pair* pr, int32_t* moving_out, int32_t* status_out,
                   int64_t* h_undecided) {
    if (!h_undecided || (a->n > 0 && !moving_out) || (a->seafloor_action == 2 && !status_out)) return -2;
    unsigned undecided = 0;
    od::SettleParams s;
    s.moving_out = moving_out;
    s.status_out = a->seafloor_action == 2 ? status_out : nullptr;
    s.undecided = &undecided;
    g_settle = &s;
    const int rc = hs2_mix(a, g, pr);
    g_settle = nullptr;
    *h_undecided = undecided;
    return rc;
}

int hs4_resuspend(int64_t n, const float* u, const float* v, float threshold, int32_t* moving, void* z, int32_t z_f64) {
    if (n < 0) return -2;
    for (int64_t i = 0; i < n; ++i) od::resuspend_one(i, u, v, threshold, moving, z, z_f64);
    return 0;
}

}
