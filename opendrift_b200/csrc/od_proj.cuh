// od_proj.cuh -- map projections of readers whose grid is not geographic, and the rotation of their vector components.
//
// The reference hands every position to pyproj (Variables.lonlat2xy, readers/basereader/variables.py:129-143) before it indexes a
// projected reader's block, and rotates x / y vector components from the grid's axes to east / north afterwards
// (rotate_vectors, :59-109: inverse projection of (x, y) and (x, y + 10 m), Geod.inv azimuth of that line, rotation by minus
// that azimuth).  Both run per particle inside the kernels here.
//
// Projections: spherical stereographic, the four aspects PROJ's stere.cpp distinguishes (Snyder 1987, eqs. 21-2..21-4,
// 20-14, 20-15, 20-18, 21-15); Mercator (7-1, 7-2 / 7-6 .. 7-9) and Lambert conformal conic with one or two standard
// parallels (15-1 .. 15-5 / 15-7 .. 15-11, 14-15, 15-9) on a sphere or an ellipsoid, organised like PROJ's merc.cpp / lcc.cpp
// (msfn, tsfn, phi2); all wrapped in PROJ's generic steps (lam = lon - lon_0 reduced to [-pi, pi], x = a x' + x_0).
// Rotated pole (+proj=ob_tran +o_proj=longlat, ob_tran.cpp o_forward / o_inverse, Snyder 5-7, 5-8b): the plane is rotated
// longitude / latitude in DEGREES, as the reference's lonlat2xy / xy2lonlat hand them out (np.degrees of what pyproj returns,
// variables.py:111-143); a = 1, x_0 = y_0 = 0 so that the generic steps leave those degrees untouched.
// Geod.inv: only the forward azimuth of a short line is needed; it is obtained by inverting the direct solution
// (mid-latitude first guess, one correction with the miss of the direct series move) -- the miss shrinks by
// (s/a)^2 ~ 2e-12 per pass for the 10 m line.
#pragma once
#include "../../include/odcuda.h"
#include "od_geod.cuh"

namespace od {

enum { PROJ_EQUIT = 0, PROJ_OBLIQ = 1, PROJ_N_POLE = 2, PROJ_S_POLE = 3 };

struct ProjStere {               // (the name is historical: kind selects the projection)
    int mode;                    // aspect of the stereographic projection
    int kind;                    // OD_PROJ_STERE_SPHERE, OD_PROJ_MERC, OD_PROJ_LCC, OD_PROJ_STERE_ELLPS, OD_PROJ_OB_TRAN
    double a, ra, akm1, sinX1, cosX1, phi0, lam0, x0, y0;   // (ob_tran: sinX1 / cosX1 of +o_lat_p)
    double e, es;                // eccentricity of the ellipsoid (0: sphere)
    double k0;                   // scale factor (Mercator: from +lat_ts or +k_0; cone: +k_0)
    double n, c, rho0;           // cone constant, F of Snyder 15-10, radius of the parallel of origin (ob_tran: n = +o_lon_p, rad)
};

constexpr double kPi = 3.14159265358979323846;
constexpr double kHalfPi = 1.57079632679489661923;
constexpr double kObTranRotDelta = 0.1;          // rotate_vectors' y-axis line on a rotated-pole plane, degrees (variables.py:79-82)

// PROJ adjlon: reduce to [-pi, pi]; values already inside are left untouched
OD_HD double adjlon(double lam) {
    if (fabs(lam) <= kPi) return lam;
    double t = lam + kPi;
    t = t - 2.0 * kPi * floor(t / (2.0 * kPi));
    return t - kPi;
}

// PROJ's pj_msfn (Snyder 14-15), pj_tsfn (15-9) and pj_phi2 (7-9)
OD_HD double proj_msfn(double sinphi, double cosphi, double es) { return cosphi / sqrt(1.0 - es * sinphi * sinphi); }
OD_HD double proj_tsfn(double phi, double sinphi, double e) {
    return tan(0.5 * (kHalfPi - phi)) / pow((1.0 - e * sinphi) / (1.0 + e * sinphi), 0.5 * e);
}
// stere.cpp's ssfn_: tan(pi/4 + phi/2) ((1 - e sin phi) / (1 + e sin phi))^(e/2); chi = 2 atan(ssfn) - pi/2 is the conformal latitude
OD_HD double proj_ssfn(double phi, double e) {
    const double s = e * sin(phi);
    return tan(0.5 * (kHalfPi + phi)) * pow((1.0 - s) / (1.0 + s), 0.5 * e);
}
OD_HD double proj_phi2(double ts, double e) {
    double phi = kHalfPi - 2.0 * atan(ts);
    for (int i = 0; i < 20; ++i) {
        const double con = e * sin(phi);
        const double nw = kHalfPi - 2.0 * atan(ts * pow((1.0 - con) / (1.0 + con), 0.5 * e));
        const double d = fabs(nw - phi);
        phi = nw;
        if (d < 1e-14) break;
    }
    return phi;
}

// The projections other than the spherical stereographic one run out of line: their code is compiled once per translation unit
// instead of once per kernel instantiation (the general step kernels alone are 36), and the kernels that only ever meet
// geographic or spherical-stereographic groups keep the size they had.  Arguments by value: no address of a kernel parameter.
struct ProjOther {
    int kind, mode;
    double e, es, k0, n, c, rho0, akm1, sinX1, cosX1;
};

OD_HD ProjOther proj_other(const ProjStere& P) {
    ProjOther q;
    q.kind = P.kind; q.mode = P.mode; q.e = P.e; q.es = P.es; q.k0 = P.k0; q.n = P.n; q.c = P.c; q.rho0 = P.rho0;
    q.akm1 = P.akm1; q.sinX1 = P.sinX1; q.cosX1 = P.cosX1;
    return q;
}

#if defined(__CUDACC__)
#define OD_PROJ_NOINLINE static __host__ __device__ __noinline__
#else
#define OD_PROJ_NOINLINE static
#endif

// lam (reduced, radians), phi (radians) -> x', y' on the unit sphere / ellipsoid (the caller applies a, x_0, y_0)
OD_PROJ_NOINLINE bool proj_forward_other(ProjOther q, double lam, double phi, double* ox, double* oy) {
    if (q.kind == OD_PROJ_MERC) {
        if (!(fabs(phi) < kHalfPi - 1e-10)) return false;
        const double py = asinh(tan(phi)) - q.e * atanh(q.e * sin(phi));
        *ox = q.k0 * lam;
        *oy = q.k0 * py;
        return true;
    }
    if (q.kind == OD_PROJ_LCC) {
        double rho;
        if (fabs(fabs(phi) - kHalfPi) < 1e-10) {
            if (!(phi * q.n > 0.0)) return false;
            rho = 0.0;
        } else {
            rho = q.es != 0.0 ? q.c * pow(proj_tsfn(phi, sin(phi), q.e), q.n) : q.c * pow(tan(kPio4 + 0.5 * phi), -q.n);
        }
        const double ln = lam * q.n;
        *ox = q.k0 * rho * sin(ln);
        *oy = q.k0 * (q.rho0 - rho * cos(ln));
        return true;
    }
    if (q.kind == OD_PROJ_STERE_ELLPS) {               // Snyder 21-24 .. 21-40 through the conformal latitude (stere.cpp: e_forward)
        double sl, cl;
        sincos(lam, &sl, &cl);
        double px, py;
        if (q.mode == PROJ_OBLIQ || q.mode == PROJ_EQUIT) {
            const double X = 2.0 * atan(proj_ssfn(phi, q.e)) - kHalfPi;
            double sX, cX;
            sincos(X, &sX, &cX);
            const double d = q.mode == PROJ_OBLIQ ? q.cosX1 * (1.0 + q.sinX1 * sX + q.cosX1 * cX * cl) : 1.0 + cX * cl;
            if (!(d > 1e-10)) return false;
            const double A = q.akm1 / d;
            px = A * cX * sl;
            py = q.mode == PROJ_OBLIQ ? A * (q.cosX1 * sX - q.sinX1 * cX * cl) : A * sX;
        } else {
            if (q.mode == PROJ_S_POLE) { phi = -phi; cl = -cl; }
            if (fabs(phi + kHalfPi) < 1e-8) return false;                  // the opposite pole
            const double rho = q.akm1 * proj_tsfn(phi, sin(phi), q.e);
            px = rho * sl;
            py = -rho * cl;
        }
        *ox = px;
        *oy = py;
        return true;
    }
    if (q.kind == OD_PROJ_OB_TRAN) {                   // ob_tran.cpp o_forward (its transverse form is the same with o_lat_p = 0)
        double sl, cl, sp, cp;
        sincos(lam, &sl, &cl);
        sincos(phi, &sp, &cp);
        const double lr = adjlon(atan2(cp * sl, q.sinX1 * cp * cl + q.cosX1 * sp) + q.n);
        const double pr = asin(fmin(1.0, fmax(-1.0, q.sinX1 * sp - q.cosX1 * cp * cl)));
        *ox = lr * kRad2Deg;
        *oy = pr * kRad2Deg;
        return true;
    }
    return false;
}

// x', y' -> lam (relative to lon_0, radians), phi (radians)
OD_PROJ_NOINLINE void proj_inverse_other(ProjOther q, double x, double y, double* olam, double* ophi) {
    if (q.kind == OD_PROJ_MERC) {
        const double ts = exp(-y / q.k0);
        const double ph = q.es != 0.0 ? proj_phi2(ts, q.e) : kHalfPi - 2.0 * atan(ts);
        *olam = x / q.k0;
        *ophi = ph;
        return;
    }
    if (q.kind == OD_PROJ_LCC) {
        x = x / q.k0;
        y = q.rho0 - y / q.k0;
        double rho = hypot(x, y);
        double ph, lm;
        if (rho != 0.0) {
            if (q.n < 0.0) { rho = -rho; x = -x; y = -y; }
            ph = q.es != 0.0 ? proj_phi2(pow(rho / q.c, 1.0 / q.n), q.e) : 2.0 * atan(pow(q.c / rho, 1.0 / q.n)) - kHalfPi;
            lm = atan2(x, y) / q.n;
        } else {
            lm = 0.0;
            ph = q.n > 0.0 ? kHalfPi : -kHalfPi;
        }
        *olam = lm;
        *ophi = ph;
        return;
    }
    if (q.kind == OD_PROJ_STERE_ELLPS) {               // stere.cpp: e_inverse (Snyder 21-36 .. 21-38, latitude by the iteration 3-4 / 7-9)
        const double rho = hypot(x, y);
        double tp, phi_l, xx, yy, halfpi, halfe;
        if (q.mode == PROJ_OBLIQ || q.mode == PROJ_EQUIT) {
            tp = 2.0 * atan2(rho * q.cosX1, q.akm1);
            double st, ct;
            sincos(tp, &st, &ct);
            phi_l = rho == 0.0 ? asin(ct * q.sinX1) : asin(fmin(1.0, fmax(-1.0, ct * q.sinX1 + y * st * q.cosX1 / rho)));
            tp = tan(0.5 * (kHalfPi + phi_l));
            xx = x * st;
            yy = rho * q.cosX1 * ct - y * q.sinX1 * st;
            halfpi = kHalfPi;
            halfe = 0.5 * q.e;
        } else {
            if (q.mode == PROJ_N_POLE) y = -y;
            tp = -rho / q.akm1;
            phi_l = kHalfPi - 2.0 * atan(-tp);
            xx = x;
            yy = y;
            halfpi = -kHalfPi;
            halfe = -0.5 * q.e;
        }
        double ph = phi_l;
        for (int i = 0; i < 20; ++i) {
            const double sp = q.e * sin(phi_l);
            ph = 2.0 * atan(tp * pow((1.0 + sp) / (1.0 - sp), halfe)) - halfpi;
            const double dd = fabs(phi_l - ph);
            phi_l = ph;
            if (dd < 1e-14) break;
        }
        if (q.mode == PROJ_S_POLE) ph = -ph;
        const double lm = (xx == 0.0 && yy == 0.0) ? 0.0 : atan2(xx, yy);
        *olam = lm;
        *ophi = ph;
        return;
    }
    if (q.kind == OD_PROJ_OB_TRAN) {                   // ob_tran.cpp o_inverse; x, y are rotated degrees
        double sl, cl, sp, cp;
        sincos(x * kDeg - q.n, &sl, &cl);
        sincos(y * kDeg, &sp, &cp);
        *ophi = asin(fmin(1.0, fmax(-1.0, q.sinX1 * sp + q.cosX1 * cp * cl)));
        *olam = atan2(cp * sl, q.sinX1 * cp * cl - q.cosX1 * sp);
        return;
    }
    *olam = 0.0;
    *ophi = 0.0;
}

// lon, lat in degrees -> x, y in metres; returns false where the projection is undefined (antipode, pole of a cylinder / cone)
OD_HD bool stere_forward(const ProjStere& P, double lon, double lat, double& x, double& y) {
    const double lam = adjlon(lon * kDeg - P.lam0);
    double phi = lat * kDeg;
    if (P.kind != OD_PROJ_STERE_SPHERE) {
        double px, py;
        if (!proj_forward_other(proj_other(P), lam, phi, &px, &py)) return false;
        x = P.a * px + P.x0;
        y = P.a * py + P.y0;
        return x == x && y == y;
    }
    double sinphi, cosphi, sinlam, coslam;
    sincos(phi, &sinphi, &cosphi);
    sincos(lam, &sinlam, &coslam);
    double px, py;
    if (P.mode == PROJ_EQUIT || P.mode == PROJ_OBLIQ) {
        const double d = P.mode == PROJ_EQUIT ? 1.0 + cosphi * coslam : 1.0 + P.sinX1 * sinphi + P.cosX1 * cosphi * coslam;
        if (!(d > 1e-10)) return false;
        const double k = P.akm1 / d;
        px = k * cosphi * sinlam;
        py = P.mode == PROJ_EQUIT ? k * sinphi : k * (P.cosX1 * sinphi - P.sinX1 * cosphi * coslam);
    } else {
        if (P.mode == PROJ_N_POLE) {
            coslam = -coslam;
            phi = -phi;
        }
        if (fabs(phi - kHalfPi) < 1e-8) return false;
        py = P.akm1 * tan(kPio4 + 0.5 * phi);
        px = sinlam * py;
        py = py * coslam;
    }
    x = P.a * px + P.x0;
    y = P.a * py + P.y0;
    return true;
}

// x, y in metres -> lon, lat in degrees
OD_HD void stere_inverse(const ProjStere& P, double x, double y, double& lon, double& lat) {
    x = (x - P.x0) * P.ra;
    y = (y - P.y0) * P.ra;
    if (P.kind != OD_PROJ_STERE_SPHERE) {
        double lm, ph;
        proj_inverse_other(proj_other(P), x, y, &lm, &ph);
        lon = adjlon(lm + P.lam0) * kRad2Deg;
        lat = ph * kRad2Deg;
        return;
    }
    const double rh = hypot(x, y);
    const double c = 2.0 * atan(rh / P.akm1);
    double sinc, cosc;
    sincos(c, &sinc, &cosc);
    const bool small = fabs(rh) <= 1e-10;
    double phi, lam = 0.0;
    if (P.mode == PROJ_EQUIT) {
        phi = small ? 0.0 : asin(fmin(1.0, fmax(-1.0, y * sinc / rh)));
        if (cosc != 0.0 || x != 0.0) lam = atan2(x * sinc, cosc * rh);
    } else if (P.mode == PROJ_OBLIQ) {
        phi = small ? P.phi0 : asin(fmin(1.0, fmax(-1.0, cosc * P.sinX1 + y * sinc * P.cosX1 / rh)));
        const double cc = cosc - P.sinX1 * sin(phi);
        if (cc != 0.0 || x != 0.0) lam = atan2(x * sinc * P.cosX1, cc * rh);
    } else {
        if (P.mode == PROJ_N_POLE) y = -y;
        phi = small ? P.phi0 : asin(P.mode == PROJ_S_POLE ? -cosc : cosc);
        lam = (x == 0.0 && y == 0.0) ? 0.0 : atan2(x, y);
    }
    lon = adjlon(lam + P.lam0) * kRad2Deg;
    lat = phi * kRad2Deg;
}

OD_HD double wrap180(double d) { return d - 360.0 * rint(d * (1.0 / 360.0)); }

// Forward azimuth (radians) at point 1 of the short WGS84 geodesic to point 2 (what rotate_vectors takes from Geod.inv)
OD_HD double inverse_azimuth_short(double lon1, double lat1, double lon2, double lat2) {
    double sm, cm;
    sincos(0.5 * (lat1 + lat2) * kDeg, &sm, &cm);
    const double w2 = 1.0 - Wgs84::e2 * sm * sm;
    const double w = sqrt(w2);
    const double M = Wgs84::a * (1.0 - Wgs84::e2) / (w2 * w);        // meridional radius of curvature
    const double Nc = Wgs84::a / w * cm;                              // radius of the parallel
    const double dlon = wrap180(lon2 - lon1);
    double north = M * (lat2 - lat1) * kDeg;
    double east = Nc * dlon * kDeg;
    // azimuth at point 1 = azimuth at the mid-point minus half the meridian convergence
    const double az = atan2(east, north) - 0.5 * dlon * kDeg * sm;
    const double s = hypot(east, north);
    double sa, ca;
    sincos(az, &sa, &ca);
    north = s * ca;
    east = s * sa;
    // one correction with the miss of the direct solution
    const SeriesStart ss = series_start(lat1);
    double lo, la;
    geod_move_ne(ss, lon1, north, east, lo, la);
    north += M * (lat2 - la) * kDeg;
    east += Nc * wrap180(lon2 - lo) * kDeg;
    return atan2(east, north);
}

// od_proj_desc (include/odcuda.h) -> the per-launch constants; the aspect and scale constant are chosen as PROJ's stere
// setup does for a sphere.  Returns 0, or 2 unknown projection, 3 bad radius / scale.
static inline int proj_from_desc(const od_proj_desc* d, ProjStere* Pp) {
    if (d->kind != OD_PROJ_STERE_SPHERE && d->kind != OD_PROJ_MERC && d->kind != OD_PROJ_LCC && d->kind != OD_PROJ_STERE_ELLPS &&
        d->kind != OD_PROJ_OB_TRAN) return 2;
    if (!(d->a > 0.0) || !(d->k_0 > 0.0)) return 3;
    ProjStere& P = *Pp;
    P.kind = d->kind;
    P.a = d->a;
    P.ra = 1.0 / d->a;
    P.phi0 = d->lat_0 * kDeg;
    P.lam0 = d->lon_0 * kDeg;
    P.x0 = d->x_0;
    P.y0 = d->y_0;
    P.es = d->kind == OD_PROJ_STERE_SPHERE ? 0.0 : d->es;           // (the sphere ignores the field)
    if (!(P.es >= 0.0 && P.es < 1.0)) return 3;
    P.e = sqrt(P.es);
    P.k0 = d->k_0;
    P.n = P.c = P.rho0 = 0.0;
    P.mode = 0;
    P.akm1 = P.sinX1 = P.cosX1 = 0.0;
    if (d->kind == OD_PROJ_OB_TRAN) {                  // ob_tran.cpp setup, new-pole form: lat_1 = +o_lat_p, lat_2 = +o_lon_p (degrees)
        if (!(fabs(d->lat_1) <= 90.0) || !(fabs(d->lat_2) <= 360.0)) return 3;
        P.a = P.ra = 1.0;                              // the plane is rotated degrees: no radius, no false origin
        P.x0 = P.y0 = 0.0;
        P.es = P.e = 0.0;
        P.k0 = 1.0;
        P.sinX1 = sin(d->lat_1 * kDeg);
        P.cosX1 = cos(d->lat_1 * kDeg);
        P.n = d->lat_2 * kDeg;
        return 0;
    }
    if (d->kind == OD_PROJ_MERC) {                     // merc.cpp: +lat_ts replaces +k_0
        if (d->has_lat_ts) {
            const double phits = fabs(d->lat_ts * kDeg);
            if (!(phits < kHalfPi)) return 3;
            P.k0 = proj_msfn(sin(phits), cos(phits), P.es);
        }
        return 0;
    }
    if (d->kind == OD_PROJ_LCC) {                      // lcc.cpp setup
        const double phi1 = d->lat_1 * kDeg, phi2 = d->lat_2 * kDeg;
        if (fabs(phi1 + phi2) < 1e-10) return 3;
        const double sinphi = sin(phi1), cosphi = cos(phi1);
        const bool secant = fabs(phi1 - phi2) >= 1e-10;
        double n = sinphi;
        if (P.es != 0.0) {
            const double m1 = proj_msfn(sinphi, cosphi, P.es), ml1 = proj_tsfn(phi1, sinphi, P.e);
            if (secant) {
                const double s2 = sin(phi2);
                n = log(m1 / proj_msfn(s2, cos(phi2), P.es)) / log(ml1 / proj_tsfn(phi2, s2, P.e));
            }
            P.c = m1 * pow(ml1, -n) / n;
            P.rho0 = fabs(fabs(P.phi0) - kHalfPi) < 1e-10 ? 0.0 : P.c * pow(proj_tsfn(P.phi0, sin(P.phi0), P.e), n);
        } else {
            if (secant) n = log(cosphi / cos(phi2)) / log(tan(kPio4 + 0.5 * phi2) / tan(kPio4 + 0.5 * phi1));
            P.c = cosphi * pow(tan(kPio4 + 0.5 * phi1), n) / n;
            P.rho0 = fabs(fabs(P.phi0) - kHalfPi) < 1e-10 ? 0.0 : P.c * pow(tan(kPio4 + 0.5 * P.phi0), -n);
        }
        P.n = n;
        if (!(n == n) || n == 0.0) return 3;
        return 0;
    }
    const double t = fabs(P.phi0);
    if (fabs(t - kHalfPi) < 1e-10) P.mode = P.phi0 < 0 ? PROJ_S_POLE : PROJ_N_POLE;
    else P.mode = t > 1e-10 ? PROJ_OBLIQ : PROJ_EQUIT;
    if (d->kind == OD_PROJ_STERE_ELLPS) {              // stere.cpp setup, ellipsoidal half
        P.es = d->es;
        if (!(P.es > 0.0 && P.es < 1.0)) return 3;
        P.e = sqrt(P.es);
        const double phits = fabs(d->has_lat_ts ? d->lat_ts * kDeg : kHalfPi);
        if (P.mode == PROJ_N_POLE || P.mode == PROJ_S_POLE) {
            if (fabs(phits - kHalfPi) < 1e-10) P.akm1 = 2.0 * d->k_0 / sqrt(pow(1.0 + P.e, 1.0 + P.e) * pow(1.0 - P.e, 1.0 - P.e));
            else P.akm1 = proj_msfn(sin(phits), cos(phits), P.es) / proj_tsfn(phits, sin(phits), P.e);
            P.sinX1 = P.cosX1 = 0.0;
        } else {
            const double sp = sin(P.phi0);
            const double X = 2.0 * atan(proj_ssfn(P.phi0, P.e)) - kHalfPi;
            P.akm1 = 2.0 * d->k_0 * cos(P.phi0) / sqrt(1.0 - P.es * sp * sp);
            P.sinX1 = sin(X);
            P.cosX1 = cos(X);
        }
        return 0;
    }
    P.sinX1 = sin(P.phi0);
    P.cosX1 = cos(P.phi0);
    const double phits = fabs(d->has_lat_ts ? d->lat_ts * kDeg : kHalfPi);
    if (P.mode == PROJ_OBLIQ || P.mode == PROJ_EQUIT) P.akm1 = 2.0 * d->k_0;
    else P.akm1 = fabs(phits - kHalfPi) >= 1e-10 ? cos(phits) / tan(kPio4 - 0.5 * phits) : 2.0 * d->k_0;
    return 0;
}

// rotate_vectors (variables.py:59-109): angle (radians) by which components along the plane's x / y axes at (px, py) are
// rotated to become east / north components.  delta is the length of the line along the y axis: 10 m on a projected plane;
// 0.1 (degrees) on a rotated-pole plane, which pyproj calls geographic (:79-82) -- the kind decides that one, so that it holds
// whatever geometry the caller built.
OD_HD double rotation_to_geographic(const ProjStere& P, double px, double py, double delta) {
    if (P.kind == OD_PROJ_OB_TRAN) delta = kObTranRotDelta;
    double lon1, lat1, lon2, lat2;
    stere_inverse(P, px, py, lon1, lat1);
    stere_inverse(P, px, py + delta, lon2, lat2);
    return -inverse_azimuth_short(lon1, lat1, lon2, lat2);
}

}  // namespace od
