// Host build of PlastDrift's device code for the CPU tests (tests/plast_host.py): plast_particle of csrc/od_plast.cuh, one loop per
// launch, with the argument checks and parameter fill of od_plast_step.  Compiled with -ffp-contract=off, as the device build rounds
// every operation on its own.
#include <math.h>
#include <stdint.h>
#include <string.h>
#include "../../opendrift_b200/csrc/od_plast.cuh"

using namespace od;

extern "C" {

int hs6_plast_step(int64_t n, double* lon, double* lat, const int32_t* moving, const void* z_in, int32_t z_f64, double* z_out,
                   const float* k, const void* tv, int32_t tv_f64, const double* rand, const int32_t* ids, unsigned long long seed, int32_t step_index,
                   const float* const* stokes, int32_t hs_mode, int32_t profile, const float* xwind, const float* ywind,
                   const void* wdf, int32_t wdf_f64, double wind_drift_depth, double dt, int32_t* h_negative) {
    if (n < 0 || !h_negative) return -2;
    *h_negative = 0;
    if (stokes && (hs_mode < 0 || hs_mode > 2 || profile < 0 || profile > 3)) return -2;
    if (n == 0) return 0;
    if (!lon || !lat || (!z_out && !z_in) || (z_out && (!k || !tv)) || (wdf && (!xwind || !ywind)) ||
        (stokes && (!stokes[0] || !stokes[1] || (hs_mode == 0 && profile != 3 && !stokes[2]))))
        return -2;
    if (stokes && profile == 3)
        for (int j = 5; j < 11; ++j)
            if (!stokes[j]) return -2;
    PlastParams p;
    memset(&p, 0, sizeof(p));
    p.n = n; p.lon = lon; p.lat = lat; p.moving = moving; p.z_in = z_in; p.z_f64 = z_f64; p.z_out = z_out;
    p.k = k; p.tv = tv; p.tv_f64 = tv_f64; p.rand = rand; p.ids = ids; p.seed = seed; p.step_index = step_index;
    if (stokes) {
        p.stokes_on = 1;
        p.st.us = stokes[0]; p.st.vs = stokes[1]; p.st.hs = stokes[2]; p.st.xwind = stokes[3]; p.st.ywind = stokes[4];
        p.st.sw_dir = stokes[5]; p.st.sw_period = stokes[6]; p.st.sw_hs = stokes[7];
        p.st.ws_dir = stokes[8]; p.st.ws_period = stokes[9]; p.st.ws_hs = stokes[10];
        p.st.hs_mode = hs_mode; p.st.profile = profile; p.st.factor = 1.0;
    }
    if (wdf) {
        p.wind_on = 1;
        p.xwind = xwind; p.ywind = ywind; p.wdf = wdf; p.wdf_f64 = wdf_f64; p.wdd = fabs(wind_drift_depth);
    }
    p.dt = dt;
    unsigned flag = 0;
    if (z_out) p.negative = &flag;
    for (int64_t i = 0; i < n; ++i) plast_particle(p, i);
    *h_negative = flag ? 1 : 0;
    return 0;
}

// the first uniform of philox_uniform2 for (seed, ids[i], step, tag): the analytical depths' stream and the mixing loop's
int hs6_philox_u0(int64_t n, unsigned long long seed, const int32_t* ids, int32_t step, uint32_t tag, double* out) {
    for (int64_t i = 0; i < n; ++i) {
        double u, spare;
        philox_uniform2(seed, (unsigned)ids[i], (unsigned)step, tag, u, spare);
        out[i] = u;
    }
    return 0;
}

}
