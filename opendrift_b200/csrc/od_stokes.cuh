// od_stokes.cuh -- Stokes drift velocity of one particle and its geodesic move.
//
// Restates PhysicsMethods.stokes_drift (opendrift/models/physics_methods.py:793-848) with the depth profiles
// stokes_drift_profile_{monochromatic,exponential,phillips} (:332-416), Hs from the environment or from wind
// (significant_wave_height, :893-906: 0.0246 |U|^2) and the wave period from wind (wave_period /
// _wave_frequency, :908-943: omega = 0.877 g / (1.17 |U|), 5 rad/s without wind), keeping NumPy's dtype flow
// (float32 environment; float32 wind speed, Hs and omega arithmetic; everything downstream float64).
// The collective decisions of the reference (is there any Stokes drift / any Hs / any wind at all) are taken by
// the host from od_minmax_f32 reductions and arrive here as hs_mode.
#pragma once
#include "od_advect.cuh"

namespace od {

struct StokesParams {
    int64_t n;
    double* lon;
    double* lat;
    const void* z;
    const float* us;
    const float* vs;
    const float* hs;
    const float* xwind;
    const float* ywind;
    const int32_t* moving;
    double dt;
    int32_t z_f64, hs_mode /* 0 env, 1 from wind, 2 constant 1 */, profile /* 0 mono, 1 exp, 2 Phillips, 3 windsea_swell */, pad_;
    // stokes_drift(factor): update_positions(stokes_u * factor, stokes_v * factor) (:843); a Python scalar or a per-element array
    double factor;
    const void* factor_arr;      // float32 / float64 (factor_f64), or NULL -> the scalar
    int32_t factor_f64, pad2_;
    // windsea_swell (:418-455): swell / wind-sea direction (degrees, 'to'), period and significant height, float32 environment
    const float* sw_dir; const float* sw_period; const float* sw_hs;
    const float* ws_dir; const float* ws_period; const float* ws_hs;
};

OD_HD double erfc_(double x) { return erfc(x); }

// ---- windsea_swell: Breivik & Christensen (2020) combined profile, in the dtype flow NumPy gives it ---------------------------------
// The environment is float32, so everything up to the depth profile is float32 arithmetic; the profile itself is float64 when the
// element depths are (z after vertical mixing, or a broadcast scalar) and float32 when z is a seeded float32 array.
OD_HD float exp_t(float x) { return expf(x); }
OD_HD double exp_t(double x) { return exp(x); }
OD_HD float sqrt_t(float x) { return sqrtf(x); }
OD_HD double sqrt_t(double x) { return sqrt(x); }
OD_HD float erfc_t(float x) { return erfcf(x); }
OD_HD double erfc_t(double x) { return erfc(x); }
OD_HD float abs_t(float x) { return fabsf(x); }
OD_HD double abs_t(double x) { return fabs(x); }
OD_HD float mul_t(float a, float b) { return OD_FMUL(a, b); }
OD_HD double mul_t(double a, double b) { return OD_DMUL(a, b); }
OD_HD float sub_t(float a, float b) { return OD_FADD(a, -b); }
OD_HD double sub_t(double a, double b) { return OD_DSUB(a, b); }

// km of stokes_transport_monochromatic (:328-330) with float32 period and height: all float32
OD_HD float transport_f32(float period, float hs) {
    const float freq = (float)(2. * 3.141592653589793) / period;
    return OD_FMUL(freq, OD_FMUL(hs, hs)) / 16.0f;
}

// stokes_drift_profile_monochromatic (:332-357): unit profile at depth z for a float32 surface drift
template <typename Z>
OD_HD Z unit_monochromatic(float speed, float period, float hs, Z z) {
    const float km = speed / OD_FMUL(2.0f, transport_f32(period, hs));
    return exp_t(mul_t((Z)OD_FMUL(2.0f, km), z));
}

// stokes_drift_profile_phillips (:387-416)
template <typename Z>
OD_HD Z unit_phillips(float speed, float period, float hs, Z z) {
    const float km = OD_FMUL(speed, (float)(1 - 2 * 1 / 3.0)) / OD_FMUL(2.0f, transport_f32(period, hs));
    const Z az = abs_t(z);
    const Z e = exp_t(mul_t((Z)OD_FMUL(2.0f, km), z));
    const Z a = sqrt_t(mul_t((Z)OD_FMUL((float)(2 * 3.141592653589793), km), az));
    const Z b = erfc_t(sqrt_t(mul_t((Z)OD_FMUL(2.0f, km), az)));
    return sub_t(e, mul_t(a, b));
}

template <typename Z>
OD_HD void windsea_swell(const StokesParams& p, int64_t i, float us, float vs, Z z, Z& su, Z& sv) {
    const float d2r = (float)3.141592653589793 / 180.0f;            // np.radians of a float32 array
    const float wsr = OD_FMUL(p.ws_dir[i], d2r), swr = OD_FMUL(p.sw_dir[i], d2r);
    const float th_ws_N = cosf(wsr), th_ws_E = sinf(wsr), th_sw_N = cosf(swr), th_sw_E = sinf(swr);
    const float sp = OD_FADD(OD_FMUL(us, th_ws_N), -OD_FMUL(vs, th_ws_E)) / OD_FADD(OD_FMUL(th_sw_E, th_ws_N), -OD_FMUL(th_sw_N, th_ws_E));
    const float swu = OD_FMUL(sp, th_sw_E), swv = OD_FMUL(sp, th_sw_N);
    const float wu = OD_FADD(us, -swu), wv = OD_FADD(vs, -swv);
    const float s_sw = sqrtf(OD_FADD(OD_FMUL(swu, swu), OD_FMUL(swv, swv)));
    const float s_w = sqrtf(OD_FADD(OD_FMUL(wu, wu), OD_FMUL(wv, wv)));
    Z au = 0, av = 0, bu = 0, bv = 0;
    if (s_sw != 0.0f) {                              // zeromask of the monochromatic part
        const Z unit = unit_monochromatic<Z>(s_sw, p.sw_period[i], p.sw_hs[i], z);
        au = mul_t((Z)swu, unit);
        av = mul_t((Z)swv, unit);
    }
    if (s_w != 0.0f) {
        const Z unit = unit_phillips<Z>(s_w, p.ws_period[i], p.ws_hs[i], z);
        bu = mul_t((Z)wu, unit);
        bv = mul_t((Z)wv, unit);
    }
    su = au + bu;
    sv = av + bv;
}

OD_HD void stokes_particle(const StokesParams& p, int64_t i) {
    const float us = p.us[i], vs = p.vs[i];
    if (p.profile == 3) {
        const double mvw = p.moving ? (double)p.moving[i] : 1.0;
        const GeodStart gw = geod_start(p.lat[i]);
        double lo, la;
        const bool f_arr64 = p.factor_arr && p.factor_f64;
        if (p.z_f64 || f_arr64) {
            double su, sv;
            if (p.z_f64) windsea_swell<double>(p, i, us, vs, ((const double*)p.z)[i], su, sv);
            else { float a, b; windsea_swell<float>(p, i, us, vs, ((const float*)p.z)[i], a, b); su = (double)a; sv = (double)b; }
            const double f = p.factor_arr ? (p.factor_f64 ? ((const double*)p.factor_arr)[i] : (double)((const float*)p.factor_arr)[i]) : p.factor;
            su = OD_DMUL(su, f);
            sv = OD_DMUL(sv, f);
            if (su == 0.0 && sv == 0.0) return;
            final_move_f64(gw, p.lon[i], su, sv, mvw, p.dt, lo, la);
        } else {                                     // float32 depths and a float32 / scalar factor: the whole chain is float32
            float su, sv;
            windsea_swell<float>(p, i, us, vs, ((const float*)p.z)[i], su, sv);
            const float f = p.factor_arr ? ((const float*)p.factor_arr)[i] : (float)p.factor;
            su = OD_FMUL(su, f);
            sv = OD_FMUL(sv, f);
            if (su == 0.0f && sv == 0.0f) return;
            final_move_f32(gw, p.lon[i], su, sv, mvw, p.dt, lo, la);
        }
        p.lon[i] = lo;
        p.lat[i] = la;
        return;
    }
    const float speed = sqrtf(OD_FADD(OD_FMUL(us, us), OD_FMUL(vs, vs)));
    if (speed == 0.0f) return;                       // zeromask: zero velocity, nothing moves
    const double z = p.z_f64 ? ((const double*)p.z)[i] : (double)((const float*)p.z)[i];
    const float xw = p.xwind ? p.xwind[i] : 0.0f, yw = p.ywind ? p.ywind[i] : 0.0f;
    const float ws = sqrtf(OD_FADD(OD_FMUL(xw, xw), OD_FMUL(yw, yw)));
    // wave period from wind (float32 quotient stored into a float64 array)
    const double omega = ws > 0.0f ? (double)((float)(0.877 * 9.81) / OD_FMUL((float)1.17, ws)) : 5.0;
    const double T = (2 * 3.141592653589793) / omega;
    const double freq = 2. * 3.141592653589793 / T;
    double hs2;                                      // np.power(Hs, 2)
    if (p.hs_mode == 0) hs2 = (double)OD_FMUL(p.hs[i], p.hs[i]);
    else if (p.hs_mode == 1) { const float h = OD_FMUL((float)0.0246, OD_FMUL(ws, ws)); hs2 = (double)OD_FMUL(h, h); }
    else hs2 = 1.0;
    const double transport = OD_DMUL(freq, hs2) / 16;
    double unit;
    if (p.profile == 0) {
        const double km = (double)speed / OD_DMUL(2.0, transport);
        unit = exp(OD_DMUL(OD_DMUL(2.0, km), z));
    } else if (p.profile == 1) {
        const double km = (double)speed / OD_DMUL(2.0, transport);
        const double ke = km / 3;
        unit = exp(OD_DMUL(OD_DMUL(2.0, ke), z)) / OD_DSUB(1.0, OD_DMUL(OD_DMUL(8.0, ke), z));
    } else {
        const double km = (double)OD_FMUL(speed, (float)(1 - 2 * 1 / 3.0)) / OD_DMUL(2.0, transport);
        const double az = fabs(z);
        unit = OD_DSUB(exp(OD_DMUL(OD_DMUL(2.0, km), z)),
                       OD_DMUL(sqrt(OD_DMUL(OD_DMUL(2 * 3.141592653589793, km), az)),
                               erfc_(sqrt(OD_DMUL(OD_DMUL(2.0, km), az)))));
    }
    double su = OD_DMUL((double)us, unit), sv = OD_DMUL((double)vs, unit);
    if (p.factor_arr || p.factor != 1.0) {           // stokes_u * factor (float64 whatever the factor's dtype)
        const double f = p.factor_arr ? (p.factor_f64 ? ((const double*)p.factor_arr)[i] : (double)((const float*)p.factor_arr)[i]) : p.factor;
        su = OD_DMUL(su, f);
        sv = OD_DMUL(sv, f);
    }
    if (su == 0.0 && sv == 0.0) return;
    const double mv = p.moving ? (double)p.moving[i] : 1.0;
    const GeodStart gs = geod_start(p.lat[i]);
    double lo, la;
    final_move_f64(gs, p.lon[i], su, sv, mv, p.dt, lo, la);
    p.lon[i] = lo;
    p.lat[i] = la;
}

// ---- drift:use_tabularised_stokes_drift: Stokes drift and Hs from the wind (physics_methods.py:488-568) ----------------------------
// wave_stokes_drift_parameterised / wave_significant_height_parameterised in the dtype flow NumPy gives them.  The wind arrives as
// fields of the reference's masked environment array, and np.ma.power squares a float32 masked array in float64 (the exponent
// becomes a 0-d int64 array, which is not a weak scalar):
//   ws = sqrt(x^2 + y^2) in float64 from the float32 wind (each square exact), ws > 30 -> 30 (NaN stays);
//   np.polyval(c, ws): y = 0*ws + c[0] is c[0] (NaN for a NaN ws), then y = y*ws + c[k] in float64;
//   us = float32(float64(x) * wf), vs likewise; Hs = float32(polyval).  No fused multiply-add anywhere.
// The coefficients are np.polyfit of the reference's tables, computed by the host.
#define OD_TAB_MAX_COEF 8

struct StokesTabParams {
    int64_t n;
    const float* xwind;
    const float* ywind;
    float* us;                   // NULL: the Stokes drift is not replaced
    float* vs;
    float* hs;                   // NULL: Hs is not replaced
    int32_t n_wf, n_hs;          // number of coefficients (polynomial order + 1)
    double wf[OD_TAB_MAX_COEF];  // highest power first, as np.polyfit returns them
    double hsc[OD_TAB_MAX_COEF];
};

OD_HD double tab_polyval(const double* c, int32_t nc, double ws) {
    if (ws != ws) return ws;
    double y = c[0];
    for (int32_t k = 1; k < nc; ++k) y = OD_DADD(OD_DMUL(y, ws), c[k]);
    return y;
}

OD_HD void stokes_tab_one(const StokesTabParams& p, int64_t i) {
    const double xw = (double)p.xwind[i], yw = (double)p.ywind[i];
    const double s2 = OD_DADD(OD_DMUL(xw, xw), OD_DMUL(yw, yw));
#if defined(__CUDA_ARCH__)
    double ws = __dsqrt_rn(s2);
#else
    double ws = sqrt(s2);
#endif
    if (ws > 30.0) ws = 30.0;
    if (p.us) {
        const double wf = tab_polyval(p.wf, p.n_wf, ws);
        p.us[i] = (float)OD_DMUL(xw, wf);
        p.vs[i] = (float)OD_DMUL(yw, wf);
    }
    if (p.hs) p.hs[i] = (float)tab_polyval(p.hsc, p.n_hs, ws);
}

}  // namespace od
