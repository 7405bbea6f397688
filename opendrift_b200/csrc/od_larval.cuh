// od_larval.cuh -- LarvalFish's per-element biology: hatching, growth and length, the egg's terminal velocity, and the larvae's
// vertical migration (opendrift/models/larvalfish.py).
//
// The reference computes these in NumPy, operation by operation in the dtypes NumPy 2 gives them.  The environment's temperature T
// and salinity S are float32; an element variable is float32 when it was seeded as an array and float64 when it was seeded as a
// scalar (promoted on release).  A Python float constant takes the dtype of the array it meets (NEP 50), a mixed float32 / float64
// operation is float64.  Here every value is carried in a double and each operation is rounded to the dtype NumPy computes it in
// (rnd): for +, -, *, / and sqrt of float32 operands the double result rounded to float32 is the float32 result.  exp, log, log10
// and pow of float32 values are the float64 functions rounded to float32 (NumPy's float32 versions are SIMD routines accurate to
// 1-3 ulp).  No fused multiply-add: every product and sum is rounded on its own.
//
// larval_develop_one, for one element (update_fish_larvae :200-231 and update_terminal_velocity :105-183):
//   (a) with p.develop: an egg (hatched == 0) adds (dt / 86400) / exp(3.65 - 0.145 T) (float32) to stage_fraction and hatches
//       (hatched = 1) at stage_fraction >= 1; a larva (hatched == 1, also one that hatched in this step) grows by Folkvord's (2005)
//       fish_growth (:185-198) in weight's dtype and gets length = exp(2.296 + 0.277 log w - 0.005128 log10(w)^2), stored in
//       length's dtype.
//   (b) with p.w_out: Sundby's (1983) terminal velocity W of every element from T, S, diameter and neutral_buoyancy_salinity: the
//       Fofonoff-Millard density of the water and of the egg (physics_methods.py:574-609), the Sharqawy viscosity (:159-178), the
//       Stokes-regime W and, where W * 1000 * d / mu > 0.5, the empirical high-Reynolds W2.  W is float64 when diameter or
//       neutral_buoyancy_salinity is, else float32.
//   Returns the flags the host's two raises need: LARVAL_STAGED (the element is an egg or a larva), LARVAL_HOT (T > 100) and
//   LARVAL_NAN_T (T is NaN: NumPy's max is then NaN and the reference does not raise).
// larval_migrate_one (larvae_vertical_migration :233-253): a larva moves to min(0, z + dir * f * swim(L) * dt), whether it is
// moving or not, with swim(L) = (0.261 L^(1.552 L^-0.08) - 5.289 / L) / 1000 in length's dtype and the sum in the wider of z's and
// length's dtypes, stored in z's dtype.
#pragma once
#include <math.h>
#include <stdint.h>
#include "od_interp.cuh"

namespace od {

#define LARVAL_STAGED 1u
#define LARVAL_HOT 2u
#define LARVAL_NAN_T 4u

struct LarvalParams {
    int64_t n;
    const float* t;              // sea_water_temperature
    const float* s;              // sea_water_salinity
    void* hatched;               // uint8 or float64 (hatched_f64)
    void* stage;                 // stage_fraction, float32 or float64 (stage_f64); likewise below
    void* weight;
    void* length;
    const void* diameter;
    const void* nbs;             // neutral_buoyancy_salinity
    void* w_out;                 // (b): terminal velocity, float64 if diameter_f64 || nbs_f64; NULL: (b) off
    void* z;                     // migration: float32 or float64 (z_f64)
    int32_t hatched_f64, stage_f64, weight_f64, length_f64, diameter_f64, nbs_f64, z_f64;
    int32_t develop;             // (a) on
    double dt;
    double swim;                 // migration: IBM:fraction_of_timestep_swimming
    double dir;                  // migration: -1 before 12:00 UTC, else +1
};

// x rounded to float32 where the operation is float32
OD_HD double lv_rnd(double x, bool f32) { return f32 ? (double)(float)x : x; }
OD_HD double lv_mul(double a, double b, bool f32) { return lv_rnd(OD_DMUL(a, b), f32); }
OD_HD double lv_add(double a, double b, bool f32) { return lv_rnd(OD_DADD(a, b), f32); }
OD_HD double lv_sub(double a, double b, bool f32) { return lv_rnd(OD_DSUB(a, b), f32); }
OD_HD double lv_div(double a, double b, bool f32) { return lv_rnd(a / b, f32); }

OD_HD double lv_load(const void* a, bool f64, int64_t i) { return f64 ? ((const double*)a)[i] : (double)((const float*)a)[i]; }
OD_HD void lv_store(void* a, bool f64, int64_t i, double v) {
    if (f64) ((double*)a)[i] = v;
    else ((float*)a)[i] = (float)v;
}

// PhysicsMethods.sea_water_density with float32 T and S of dtype float32 (s32) or float64
OD_HD double lv_density(double t, double s, bool s32) {
    const bool F = true;
    double r1 = lv_add(lv_mul(lv_rnd(6.536332E-09, F), t, F), -lv_rnd(1.120083E-06, F), F);
    r1 = lv_add(lv_mul(r1, t, F), lv_rnd(1.001685E-04, F), F);
    r1 = lv_sub(lv_mul(r1, t, F), lv_rnd(9.095290E-03, F), F);
    r1 = lv_add(lv_mul(r1, t, F), lv_rnd(6.793952E-02, F), F);
    r1 = lv_sub(lv_mul(r1, t, F), lv_rnd(28.263737, F), F);
    double r2 = lv_sub(lv_mul(lv_rnd(5.3875E-09, F), t, F), lv_rnd(8.2467E-07, F), F);
    r2 = lv_add(lv_mul(r2, t, F), lv_rnd(7.6438E-05, F), F);
    r2 = lv_sub(lv_mul(r2, t, F), lv_rnd(4.0899E-03, F), F);
    r2 = lv_add(lv_mul(r2, t, F), lv_rnd(8.24493E-01, F), F);
    double r3 = lv_add(lv_mul(-lv_rnd(1.6546E-06, F), t, F), lv_rnd(1.0227E-04, F), F);
    r3 = lv_sub(lv_mul(r3, t, F), lv_rnd(5.72466E-03, F), F);
    // SIG = R1 + (R4*S + R3*sqrt(S) + R2)*S, in S's dtype from the first product on
    double q = lv_add(lv_mul(lv_rnd(4.8314E-04, s32), s, s32), lv_mul(r3, lv_rnd(sqrt(s), s32), s32), s32);
    q = lv_mul(lv_add(q, r2, s32), s, s32);
    const double sig = lv_add(r1, q, s32);
    return lv_add(lv_add(sig, lv_rnd(28.106331, s32), s32), lv_rnd(1000., s32), s32);
}

// seawater_dynamic_viscosity (Sharqawy et al. 2010) of float32 T and S, float32
OD_HD double lv_viscosity(double t, double s) {
    const bool F = true;
    const double tp = lv_add(t, lv_rnd(64.993, F), F);
    const double mu_w = lv_add(lv_rnd(4.2844e-5, F),
                               lv_div(1.0, lv_sub(lv_mul(lv_rnd(0.157, F), lv_mul(tp, tp, F), F), lv_rnd(91.296, F), F), F), F);
    const double t2 = lv_mul(t, t, F);
    const double a = lv_sub(lv_add(lv_rnd(1.541, F), lv_mul(lv_rnd(1.998e-2, F), t, F), F), lv_mul(lv_rnd(9.52e-5, F), t2, F), F);
    const double b = lv_add(lv_sub(lv_rnd(7.974, F), lv_mul(lv_rnd(7.561e-2, F), t, F), F), lv_mul(lv_rnd(4.724e-4, F), t2, F), F);
    const double sk = lv_div(s, lv_rnd(1000., F), F);
    const double c = lv_add(lv_add(1.0, lv_mul(a, sk, F), F), lv_mul(b, lv_mul(sk, sk, F), F), F);
    return lv_mul(mu_w, c, F);
}

// (b) the terminal velocity of one element
OD_HD double lv_velocity(double t, double s, double d, double sal, bool d32, bool sal32) {
    const bool F = true;
    const bool w32 = d32 && sal32;                      // W's dtype
    const double dens_w = lv_density(t, s, true);
    const double dens_e = lv_density(t, sal, sal32);
    const double dr = lv_sub(dens_w, dens_e, sal32);     // float32 - dtype(sal)
    const double mu = lv_viscosity(t, s);
    const double g = 9.81;
    // W = (1.0 / mu) * (1.0 / 18.0) * g * d ** 2 * dr
    double w = lv_mul(lv_mul(lv_div(1.0, mu, F), lv_rnd(1.0 / 18.0, F), F), lv_rnd(g, F), F);
    w = lv_mul(lv_mul(w, lv_mul(d, d, d32), d32), dr, w32);
    // W * 1000 * d / mu > 0.5
    const double re = lv_div(lv_mul(lv_mul(w, 1000., w32), d, w32), mu, w32);
    if (!(re > 0.5)) return w;
    // the high Reynolds number regime, lengths in cm
    const double mu2 = lv_mul(lv_rnd(0.01854, F), lv_rnd(exp(lv_mul(-lv_rnd(0.02783, F), t, F)), F), F);
    double x = lv_div(lv_mul(lv_rnd(9.0, F), lv_mul(mu2, mu2, F), F), lv_rnd(100 * g, F), F);
    x = lv_div(lv_mul(x, dens_w, F), dr, sal32);
    const double cube = lv_rnd(pow(x, lv_rnd(1.0 / 3.0, sal32)), sal32);
    const double d0 = lv_sub(lv_mul(d, lv_rnd(100., d32), d32), lv_mul(lv_rnd(0.4, sal32), cube, sal32), w32);
    const double p1 = lv_rnd(pow(lv_mul(lv_rnd(0.001, sal32), dr, sal32), lv_rnd(2.0 / 3.0, sal32)), sal32);
    const double p2 = lv_rnd(pow(lv_mul(lv_mul(mu2, lv_rnd(0.001, F), F), dens_w, F), lv_rnd(-1.0 / 3.0, F)), F);
    const double w2 = lv_mul(lv_mul(lv_mul(lv_rnd(19.0, w32), d0, w32), p1, w32), p2, w32);
    return lv_div(w2, lv_rnd(100., w32), w32);
}

// fish_growth (:185-198): the weight gained by a larva of weight w (dtype: w32) at float32 temperature t in dt seconds
OD_HD double lv_growth(double w, double t, bool w32, double dt) {
    const bool F = true;
    const double lw = lv_rnd(log(w), w32);
    double gr = lv_add(lv_rnd(1.08, F), lv_mul(lv_rnd(1.79, F), t, F), F);
    gr = lv_sub(gr, lv_mul(lv_mul(lv_rnd(0.074, F), t, F), lw, w32), w32);
    gr = lv_sub(gr, lv_mul(lv_mul(lv_rnd(0.0965, F), t, F), lv_mul(lw, lw, w32), w32), w32);
    gr = lv_add(gr, lv_mul(lv_mul(lv_rnd(0.0112, F), t, F), lv_rnd(pow(lw, 3.0), w32), w32), w32);
    // g = log(GR / 100 + 1) * dt / 86400, left to right
    double g = lv_rnd(log(lv_add(lv_div(gr, 100., w32), 1.0, w32)), w32);
    g = lv_div(lv_mul(g, lv_rnd(dt, w32), w32), lv_rnd(86400., w32), w32);
    return lv_mul(w, lv_sub(lv_rnd(exp(g), w32), 1.0, w32), w32);
}

OD_HD unsigned larval_develop_one(const LarvalParams& p, int64_t i) {
    const bool F = true;
    const double t = (double)p.t[i];
    unsigned flags = (t != t) ? LARVAL_NAN_T : (t > 100.0 ? LARVAL_HOT : 0u);
    if (p.develop) {
        double h = p.hatched_f64 ? ((const double*)p.hatched)[i] : (double)((const uint8_t*)p.hatched)[i];
        if (h == 0.0) {
            flags |= LARVAL_STAGED;
            const double dur = lv_rnd(exp(lv_sub(lv_rnd(3.65, F), lv_mul(lv_rnd(0.145, F), t, F), F)), F);
            const double frac = lv_div(lv_rnd(p.dt / 86400., F), dur, F);
            const double sf = lv_add(lv_load(p.stage, p.stage_f64, i), frac, !p.stage_f64);
            lv_store(p.stage, p.stage_f64, i, sf);
            if (sf >= 1.0) {
                h = 1.0;
                if (p.hatched_f64) ((double*)p.hatched)[i] = 1.0;
                else ((uint8_t*)p.hatched)[i] = 1;
            }
        }
        if (h == 1.0) {
            flags |= LARVAL_STAGED;
            const bool w32 = !p.weight_f64;
            double w = lv_load(p.weight, p.weight_f64, i);
            w = lv_add(w, lv_growth(w, t, w32, p.dt), w32);
            lv_store(p.weight, p.weight_f64, i, w);
            const double l10 = lv_rnd(log10(w), w32);
            double e = lv_add(lv_rnd(2.296, w32), lv_mul(lv_rnd(0.277, w32), lv_rnd(log(w), w32), w32), w32);
            e = lv_sub(e, lv_mul(lv_rnd(0.005128, w32), lv_mul(l10, l10, w32), w32), w32);
            lv_store(p.length, p.length_f64, i, lv_rnd(exp(e), w32));
        }
    }
    if (p.w_out) {
        const double w = lv_velocity(t, (double)p.s[i], lv_load(p.diameter, p.diameter_f64, i), lv_load(p.nbs, p.nbs_f64, i),
                                     !p.diameter_f64, !p.nbs_f64);
        lv_store(p.w_out, p.diameter_f64 || p.nbs_f64, i, w);
    }
    return flags;
}

OD_HD void larval_migrate_one(const LarvalParams& p, int64_t i) {
    const double h = p.hatched_f64 ? ((const double*)p.hatched)[i] : (double)((const uint8_t*)p.hatched)[i];
    if (h != 1.0) return;
    const bool l32 = !p.length_f64;
    const double len = lv_load(p.length, p.length_f64, i);
    const double ex = lv_mul(lv_rnd(1.552, l32), lv_rnd(pow(len, lv_rnd(-0.08, l32)), l32), l32);
    double sw = lv_sub(lv_mul(lv_rnd(0.261, l32), lv_rnd(pow(len, ex), l32), l32), lv_div(lv_rnd(5.289, l32), len, l32), l32);
    sw = lv_div(sw, lv_rnd(1000., l32), l32);
    const double m = lv_mul(lv_mul(lv_rnd(p.swim, l32), sw, l32), lv_rnd(p.dt, l32), l32);
    const bool s32 = l32 && !p.z_f64;                  // the sum's dtype
    const double v = lv_add(lv_load(p.z, p.z_f64, i), lv_mul(p.dir, m, l32), s32);
    lv_store(p.z, p.z_f64, i, 0.0 < v ? 0.0 : v);      // np.minimum(0, v): v where equal (-0.0) or NaN
}

}  // namespace od
