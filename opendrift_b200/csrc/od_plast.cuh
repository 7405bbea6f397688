// od_plast.cuh -- PlastDrift's step after the current move, for one element: submerging, Stokes drift and wind drift.
//
// Restates, in the reference's order (opendrift/models/plastdrift.py:80-107):
//   (a) update_particle_depth with vertical_mixing:mixingmodel = 'analytical' (:102-107):
//         z = -np.random.exponential(scale=K / terminal_velocity, size=n)
//       K is the float32 environment; the scale is float32 with a float32 terminal velocity (an array the user seeded) and float64
//       with a float64 one (a scalar, promoted by LagrangianArray.move_elements).  NumPy's legacy exponential is
//       scale * standard_exponential(), so z = -(double(scale) * E) in float64, for every active element (moving or not).  E is the
//       host's np.random.standard_exponential(n) (bit parity) or -log(1 - u) with u from Philox keyed by (seed, ID, step, tag).
//       NumPy raises ValueError('scale < 0') for any non-NaN scale whose sign bit is set (-0.0 and -inf included): such an element
//       raises the negative flag, and the host raises before the new depths are used.
//   (b) stokes_drift (physics_methods.py:793-848) at the new depth: stokes_particle of od_stokes.cuh, unchanged.
//   (c) advect_wind (physics_methods.py:712-791) at the new depth, in the dtype flow of the advect_wind helper:
//         wind_drift_depth != 0:  w = wdf * (|wdd| + z) / |wdd| in float64, wdf above the surface (z > 0), 0 below -|wdd|;
//                                 update_positions(x_wind * w, y_wind * w) in float64
//         wind_drift_depth == 0:  w = wdf where z >= 0, else 0, in wdf's dtype; update_positions in that dtype
//       (wind_drift_factor is float32 when seeded as an array, float64 when seeded as a scalar).
// No fused multiply-add: every product and sum is rounded on its own (OD_DMUL / OD_FMUL / OD_DADD / OD_DSUB).
#pragma once
#include "od_mix.cuh"
#include "od_stokes.cuh"

namespace od {

// the Philox stream of the analytical depths: distinct from the mixing loop's (iteration numbers) and Leeway's tags
#define OD_PLAST_TAG 0x504c4153u

struct PlastParams {
    int64_t n;
    double* lon;
    double* lat;
    const int32_t* moving;       // NULL: all move
    const void* z_in;            // float32 or float64 (z_f64): the depth when (a) is off
    double* z_out;               // (a): the new float64 depths; NULL: (a) off
    const float* k;              // (a): ocean_vertical_diffusivity, float32
    const void* tv;              // (a): terminal_velocity, float32 or float64 (tv_f64)
    const double* rand;          // (a): standard exponential draws; NULL: Philox
    const int32_t* ids;          // (a, Philox): element IDs (NULL: the index)
    unsigned* negative;          // (a): set to 1 where a scale is negative
    unsigned long long seed;
    int32_t step_index, z_f64, tv_f64, wdf_f64, stokes_on, wind_on;
    StokesParams st;             // (b): n, lon, lat, z, z_f64 are filled per element
    const float* xwind;          // (c)
    const float* ywind;
    const void* wdf;             // float32 or float64 (wdf_f64)
    double wdd;                  // |drift:wind_drift_depth|
    double dt;
};

// (a): the new depth of element i, float64
OD_HD double plast_depth(const PlastParams& p, int64_t i) {
    double scale;
    if (p.tv_f64) scale = (double)p.k[i] / ((const double*)p.tv)[i];
    else scale = (double)(p.k[i] / ((const float*)p.tv)[i]);
    if (signbit(scale) && !(scale != scale)) *p.negative = 1u;
    double e;
    if (p.rand) {
        e = p.rand[i];
    } else {
        double u, spare;
        philox_uniform2(p.seed, p.ids ? (unsigned)p.ids[i] : (unsigned)i, (unsigned)p.step_index, OD_PLAST_TAG, u, spare);
        e = -log(OD_DSUB(1.0, u));
    }
    return -OD_DMUL(scale, e);
}

// (c) at depth z (Z: float or double, the depth array's dtype)
template <typename Z>
OD_HD void plast_wind(const PlastParams& p, int64_t i, Z z) {
    const double mv = p.moving ? (double)p.moving[i] : 1.0;
    const GeodStart gs = geod_start(p.lat[i]);
    double lo, la;
    const double wdf = p.wdf_f64 ? ((const double*)p.wdf)[i] : (double)((const float*)p.wdf)[i];
    if (p.wdd != 0.0) {
        double w = 0.0;
        if ((double)z >= -p.wdd) w = (double)z > 0.0 ? wdf : OD_DMUL(wdf, OD_DADD(p.wdd, (double)z)) / p.wdd;
        final_move_f64(gs, p.lon[i], OD_DMUL((double)p.xwind[i], w), OD_DMUL((double)p.ywind[i], w), mv, p.dt, lo, la);
    } else if (p.wdf_f64) {
        const double w = z >= (Z)0 ? wdf : 0.0;
        final_move_f64(gs, p.lon[i], OD_DMUL((double)p.xwind[i], w), OD_DMUL((double)p.ywind[i], w), mv, p.dt, lo, la);
    } else {
        const float w = z >= (Z)0 ? ((const float*)p.wdf)[i] : 0.0f;
        final_move_f32(gs, p.lon[i], OD_FMUL(p.xwind[i], w), OD_FMUL(p.ywind[i], w), mv, p.dt, lo, la);
    }
    p.lon[i] = lo;
    p.lat[i] = la;
}

OD_HD void plast_particle(const PlastParams& p, int64_t i) {
    const void* zp = p.z_in;
    int32_t z_f64 = p.z_f64;
    if (p.z_out) {
        p.z_out[i] = plast_depth(p, i);
        zp = p.z_out;
        z_f64 = 1;
    }
    if (p.stokes_on) {
        StokesParams s = p.st;
        s.n = p.n; s.lon = p.lon; s.lat = p.lat; s.z = zp; s.z_f64 = z_f64; s.moving = p.moving; s.dt = p.dt;
        stokes_particle(s, i);
    }
    if (p.wind_on) {
        if (z_f64) plast_wind<double>(p, i, ((const double*)zp)[i]);
        else plast_wind<float>(p, i, ((const float*)zp)[i]);
    }
}

}  // namespace od
