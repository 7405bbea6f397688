// od_ship.cuh -- one ShipDrift time step of one ship.
//
// Restates ShipDrift.update (opendrift/models/shipdrift.py:216-343) once the start-of-step environment is known: the current move
// (update_positions of the float32 current), the wind force, the 100-point wave spectrum (recomputed per frequency, never stored),
// the trapezoid sums of the wave drift force F and the wave damping beta2 with the wforce.dat table below 7 rad/s, the long- and
// medium-period factors, the form drag, the wave direction (wind or Stokes drift, decided on the host over the whole array), the four
// iterations of the force balance, the ship move, and the stranding flag (land_binary_mask == 1 at the start-of-step position).
//
// Every operation follows the dtype NumPy 2 (NEP 50) gives it in the reference: float32 where float32 arrays meet Python scalars,
// float64 where an array is float64.  Products and sums go through the explicit-rounding macros (no FMA contraction).  NumPy's
// float32 power / exp / arctan2 are SIMD implementations accurate to 1-2.3 ulp; here they are the float64 functions rounded to
// float32, so a spectrum value can differ from the reference's by an ulp or two (about 1e-7 relative, well under a millimetre of
// ship move per hour).
//
// The table lookup reproduces scipy's LinearNDInterpolator on the (omega, beam/length, draft/length) grid bit for bit: every
// non-degenerate tetrahedron of the Delaunay triangulation lies in one grid box; the query takes the first tetrahedron of its box (in
// the triangulation's order) whose barycentric coordinates are all >= -100 DBL_EPSILON and evaluates scipy's formula in scipy's order.
#pragma once
#include <float.h>
#include "od_advect.cuh"

namespace od {

// table layout (built by models/shipdrift.py): wtab = omega[nomega] | BL[nbeam] | DL[ndraft] | per tetrahedron 20 doubles
// (transform rows T[3][3], offset r[3], F at the 4 vertices, D at the 4 vertices); wbox[box .. box + 1] is the range of the box's
// tetrahedra, box = (i_omega * (nbeam - 1) + i_beam) * (ndraft - 1) + i_draft.
#define OD_SHIP_TET 20

struct ShipParams {
    int64_t n;
    double* lon;
    double* lat;
    int32_t* moving;                  // NULL: all moving; set to 0 where a ship strands
    int32_t* status;                  // NULL: no stranding flag
    const float* length; const float* height; const float* draft; const float* beam;
    const float* cf; const float* cd;
    const uint8_t* orientation;
    const float* cu; const float* cv; const float* xw; const float* yw;
    float* hs;                        // read, or (hs_wind) written: 0.0246 ws^2
    float* tm;                        // the reader's period (Tm02 or Tp), or (tm_wind) written: the period from the wind
    const float* sx; const float* sy; // NULL: wave direction from the wind
    const float* mask;                // NULL: no stranding
    const double* wtab;
    const int32_t* wbox;
    unsigned* stranded;               // set to 1 when a ship strands (may be NULL)
    double dt;
    float tm_fill;                    // replaces T == 0 (np.mean(T[T > 0])) when tm_fill_on
    int32_t nomega, nbeam, ndraft;
    int32_t hs_wind, tm_wind, tm_fill_on, strand_code;
};

OD_HD float ship_clip(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }

// np.searchsorted(ax, x, 'right') - 1 clamped to the boxes
OD_HD int ship_cell(const double* ax, int n, double x) {
    int k = -1;
    for (int j = 0; j < n; ++j) k += ax[j] <= x ? 1 : 0;
    return k < 0 ? 0 : (k > n - 2 ? n - 2 : k);
}

// LinearNDInterpolator of F and D at (x0, x1, x2) inside box `box` (one lookup serves both: they share the triangulation)
OD_HD void ship_wforce(const ShipParams& p, int box, double x0, double x1, double x2, double& f, double& d) {
    const double* tets = p.wtab + p.nomega + p.nbeam + p.ndraft;
    const double eps = 100.0 * DBL_EPSILON;
    f = d = NAN;
    for (int k = p.wbox[box]; k < p.wbox[box + 1]; ++k) {
        const double* t = tets + (int64_t)k * OD_SHIP_TET;
        const double y[3] = {OD_DSUB(x0, t[9]), OD_DSUB(x1, t[10]), OD_DSUB(x2, t[11])};
        double c[4];
        c[3] = 1.0;
        for (int i = 0; i < 3; ++i) {
            double ci = 0.0;
            for (int j = 0; j < 3; ++j) ci = OD_DADD(ci, OD_DMUL(t[3 * i + j], y[j]));
            c[i] = ci;
            c[3] = OD_DSUB(c[3], ci);
        }
        if (!(c[0] >= -eps && c[1] >= -eps && c[2] >= -eps && c[3] >= -eps)) continue;
        double vf = 0.0, vd = 0.0;
        for (int j = 0; j < 4; ++j) {
            vf = OD_DADD(vf, OD_DMUL(c[j], t[12 + j]));
            vd = OD_DADD(vd, OD_DMUL(c[j], t[16 + j]));
        }
        f = vf;
        d = vd;
        return;
    }
}

// float32 x^k, k = 4 or 5: the float64 product rounded once to float32
OD_HD float ship_pow4f(float x) { const double x2 = OD_DMUL((double)x, (double)x); return (float)OD_DMUL(x2, x2); }
OD_HD float ship_pow5f(float x) {
    const double x2 = OD_DMUL((double)x, (double)x);
    return (float)OD_DMUL(OD_DMUL(x2, x2), (double)x);
}

// the ship's move velocity (u, v) in float64 from the forces; also the wave period and Hs as the reference obtains them
OD_HD void ship_velocity(const ShipParams& p, int64_t i, double& vel_u, double& vel_v) {
    const float xw = p.xw[i], yw = p.yw[i];
    const float ws = sqrtf(OD_FADD(OD_FMUL(xw, xw), OD_FMUL(yw, yw)));      // wind_speed(): float32
    // wave_period() (physics_methods.py:918-943): a reader's float32 period (zeros replaced by the mean), or from the wind in float64
    double Td;
    float Tf = 0.0f;
    const bool t64 = p.tm_wind != 0;
    if (t64) {
        const double omega = ws > 0.0f ? (double)((float)(0.877 * 9.81) / OD_FMUL(1.17f, ws)) : 5.0;
        Td = (2.0 * 3.141592653589793) / omega;
        p.tm[i] = (float)Td;                                                   // written back into the environment (float32)
    } else {
        Tf = p.tm[i];
        if (p.tm_fill_on && Tf == 0.0f) Tf = p.tm_fill;
        Td = (double)Tf;
    }
    // significant_wave_height(): the reader's, or 0.0246 ws^2 in float32 (written back into the environment)
    float Hs;
    if (p.hs_wind) {
        Hs = OD_FMUL(0.0246f, OD_FMUL(ws, ws));
        p.hs[i] = Hs;
    } else {
        Hs = p.hs[i];
    }
    const float L = p.length[i];
    float bl = p.beam[i] / L, dl = p.draft[i] / L;
    bl = ship_clip(ship_clip(bl, 0.12f, 0.18f), 0.121f, 0.179f);
    dl = ship_clip(ship_clip(dl, 0.025f, 0.07f), 0.0251f, 0.069f);
    const float exposed = OD_FADD(p.height[i], -p.draft[i]);
    const float area_dry = OD_FMUL(L, exposed), area_wet = OD_FMUL(L, p.draft[i]);
    // wind force (float32)
    const float F_wind = OD_FMUL(OD_FMUL(OD_FMUL(0.625f, p.cf[i]), area_dry), OD_FMUL(ws, ws));
    float Fwx = OD_FMUL(F_wind, xw) / ws, Fwy = OD_FMUL(F_wind, yw) / ws;
    if (ws == 0.0f) Fwx = Fwy = 0.0f;
    // wave spectrum parameters
    const float scale1 = sqrtf(9.81f / L);
    double d64 = 0.0, b64 = 0.0;
    float d32 = 0.0f, b32 = 0.0f;
    if (t64) {
        const double w = (2.0 * 3.141592653589793) / Td;
        const double tmp = pow(w, 4.0);
        d64 = OD_DMUL(OD_DMUL(tmp, (double)Hs), (double)Hs) / (4.0 * 3.141592653589793);
        b64 = tmp / 3.141592653589793;
    } else {
        const float tmp = ship_pow4f((float)(2.0 * 3.141592653589793) / Tf);
        d32 = OD_FMUL(OD_FMUL(tmp, Hs), Hs) / (float)(4.0 * 3.141592653589793);
        b32 = tmp / (float)3.141592653589793;
    }
    const double dom = (12.0 - 2.25) / 99;
    const int bb = ship_cell(p.wtab + p.nomega, p.nbeam, (double)bl);
    const int bd = ship_cell(p.wtab + p.nomega + p.nbeam, p.ndraft, (double)dl);
    double F = 0.0, B = 0.0;
    double f1, d1, f2 = 0.0, d2 = 0.0;
    bool a1, a2 = false;                 // f1 / f2 are interpolator arrays (float64) rather than Python floats
    for (int k = 0; k < 100; ++k) {
        const double omi0 = OD_DADD(2.25, OD_DMUL((double)k, dom));
        f1 = f2; d1 = d2; a1 = a2;
        if (omi0 < 7.0) {
            const int bo = ship_cell(p.wtab, p.nomega, omi0);
            ship_wforce(p, (bo * (p.nbeam - 1) + bb) * (p.ndraft - 1) + bd, omi0, (double)bl, (double)dl, f2, d2);
            a2 = true;
        } else {
            f2 = 0.5;
            d2 = OD_DMUL(OD_DMUL(4.0, omi0), 0.5);
            a2 = false;
        }
        // s[k] = d * exp(-b / omi^4) / omi^5, omi = omi0 * scale1 in float32
        const float omi = OD_FMUL((float)omi0, scale1);
        double s;
        if (t64) {
            s = OD_DMUL(d64, exp(-b64 / (double)ship_pow4f(omi))) / (double)ship_pow5f(omi);
        } else {
            const float e = (float)exp((double)(-b32 / ship_pow4f(omi)));
            s = (double)(OD_FMUL(d32, e) / ship_pow5f(omi));
        }
        const double s2 = OD_DMUL(s, s);
        const double cF = OD_DMUL(OD_DMUL(0.5, OD_DADD(f1, f2)), dom);
        const double cD = OD_DMUL(OD_DMUL(0.5, OD_DADD(d1, d2)), dom);
        double tF, tD;
        if (a1 || a2) {
            tF = OD_DMUL(OD_DMUL(cF, (double)scale1), s2);
            tD = OD_DMUL(OD_DMUL(cD, (double)scale1), s2);
        } else {                         // Python float * float32 array: float32
            tF = OD_DMUL((double)OD_FMUL((float)cF, scale1), s2);
            tD = OD_DMUL((double)OD_FMUL((float)cD, scale1), s2);
        }
        F = OD_DADD(F, tF);
        B = OD_DADD(B, tD);
    }
    F = OD_DMUL(OD_DMUL(OD_DMUL(F, 1025.0), 9.81), (double)L);
    B = OD_DMUL(OD_DMUL(B, 1025.0), (double)sqrtf(OD_FMUL(9.81f, L)));
    // long and medium periods: compared in the period's dtype
    if (t64) {
        if (Td > 8.55) {
            F = OD_DMUL(F, 0.66);
            B = OD_DMUL(B, 0.60);
        }
        if (Td >= 5.7 && Td <= 8.55) {
            const double x = OD_DSUB(Td, 5.7);
            F = OD_DMUL(F, OD_DSUB(1.0, OD_DMUL(0.34, x) / 2.85));
            B = OD_DMUL(B, OD_DSUB(1.0, OD_DMUL(0.4, x) / 2.85));
        }
    } else {
        if (Tf > 8.55f) {
            F = OD_DMUL(F, 0.66);
            B = OD_DMUL(B, 0.60);
        }
        if (Tf >= 5.7f && Tf <= 8.55f) {
            const float x = OD_FADD(Tf, -5.7f);
            F = OD_DMUL(F, (double)OD_FADD(1.0f, -(OD_FMUL(0.34f, x) / 2.85f)));
            B = OD_DMUL(B, (double)OD_FADD(1.0f, -(OD_FMUL(0.4f, x) / 2.85f)));
        }
    }
    // form drag (float32) and the wave direction (float64: radians(offset) + float32 arctan2)
    const float beta1 = OD_FMUL(OD_FMUL(512.5f, p.cd[i]), area_wet);
    const double offset = OD_DMUL(-40.0, OD_DSUB((double)p.orientation[i], 0.5));
    const float ang = p.sx ? (float)atan2((double)p.sy[i], (double)p.sx[i]) : (float)atan2((double)yw, (double)xw);
    const double wave_dir = OD_DADD(OD_DMUL(offset, 3.141592653589793 / 180.0), (double)ang);
    const double cw = cos(wave_dir), sw = sin(wave_dir);
    const double Fx = OD_DADD((double)Fwx, OD_DMUL(F, cw)), Fy = OD_DADD((double)Fwy, OD_DMUL(F, sw));
    const double F_total = sqrt(OD_DADD(OD_DMUL(Fx, Fx), OD_DMUL(Fy, Fy)));
    const double b1x2 = (double)OD_FMUL(2.0f, beta1), b1x4 = (double)OD_FMUL(4.0f, beta1);
    double uw_tot = 0.0, uw_dir = 0.0;
    for (int it = 0; it < 4; ++it) {
        const double f2x = OD_DMUL(OD_DMUL(B, uw_tot), cw), f2y = OD_DMUL(OD_DMUL(B, uw_tot), sw);
        uw_dir = atan2(OD_DSUB(Fy, f2y), OD_DSUB(Fx, f2x));
        const double bet2c = OD_DMUL(B, cos(OD_DSUB(wave_dir, uw_dir)));
        uw_tot = OD_DADD(-bet2c / b1x2, sqrt(OD_DADD(OD_DMUL(bet2c, bet2c), OD_DMUL(b1x4, F_total))) / b1x2);
    }
    vel_u = OD_DMUL(uw_tot, cos(uw_dir));
    vel_v = OD_DMUL(uw_tot, sin(uw_dir));
}

OD_HD void ship_particle(const ShipParams& p, int64_t i) {
    const double mv = p.moving ? (double)p.moving[i] : 1.0;
    double u, v;
    ship_velocity(p, i, u, v);
    double lon1, lat1;
    final_move_f32(geod_start(p.lat[i]), p.lon[i], p.cu[i], p.cv[i], mv, p.dt, lon1, lat1);   // update_positions(current)
    final_move_f64(geod_start(lat1), lon1, u, v, mv, p.dt, lon1, lat1);                       // update_positions(ship velocity)
    p.lon[i] = lon1;
    p.lat[i] = lat1;
    if (p.mask && p.status && p.mask[i] == 1.0f) {                 // deactivate_elements(land_binary_mask == 1, 'ship stranded')
        if (p.status[i] == 0) p.status[i] = p.strand_code;
        if (p.moving) p.moving[i] = 0;
        if (p.stranded) *p.stranded = 1u;
    }
}

}  // namespace od
