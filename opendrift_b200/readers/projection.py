"""Host-side map projection of a reader's native plane, for the handful of points user scripts convert
(`reader.xy2lonlat(x, y)` to place seeds, `reader.lonlat2xy(lon, lat)` to read results back: BaseReader.xy2lonlat /
lonlat2xy, opendrift/readers/basereader/variables.py:114-143, which wrap pyproj.Proj).  The per-particle projection of
the hot path runs on the device (csrc/od_analytic.cuh: stere_forward / stere_inverse); this module only parses the
proj4 string into the library's od_proj_desc and mirrors the same closed forms in NumPy for those few host points.

Supported: '+proj=stere' on a sphere ('+R=...' or '+a=... +e=0') or an ellipsoid, all four aspects (Snyder 1987, ch. 21);
'+proj=merc' and '+proj=lcc' (one or two standard parallels) on a sphere or an ellipsoid (Snyder ch. 7 and 15; PROJ's merc.cpp /
lcc.cpp); the rotated pole '+proj=ob_tran +o_proj=longlat +o_lat_p=.. [+o_lon_p=..] +lon_0=..', whose plane is rotated degrees.
"""
import re

import numpy as np

from .. import _lib

_DEG = np.pi / 180.0


def parse_proj4(s):
    out = {}
    for m in re.finditer(r'\+([A-Za-z_0-9]+)(?:=(\S+))?', str(s)):
        k, v = m.group(1), m.group(2)
        if v is None:
            out[k] = True
        else:
            try:
                out[k] = float(v)
            except ValueError:
                out[k] = v
    return out


def is_geographic(proj4):
    """A plain longitude / latitude grid.  A rotated pole (+proj=ob_tran +o_proj=longlat) is not one: its axes are rotated."""
    if is_rotated_pole(proj4):
        return False
    return any(k in str(proj4) for k in ('latlong', 'longlat', 'lonlat', 'latlon'))


class SphericalStereographic:
    def __init__(self, proj4):
        p = parse_proj4(proj4)
        if p.get('proj') != 'stere':
            raise NotImplementedError('projected readers on the GPU path: spherical +proj=stere only; got %s' % proj4)
        if 'R' in p:
            a = float(p['R'])
        else:
            a = float(p.get('a', 6378137.0))
            es = float(p['e']) ** 2 if 'e' in p else float(p.get('es', 0.0))
            if es != 0.0 or any(k in p for k in ('rf', 'f', 'ellps', 'datum')) or ('b' in p and float(p['b']) != a):
                raise NotImplementedError('ellipsoidal stereographic is not on the GPU path: %s' % proj4)
        if p.get('units', 'm') != 'm':
            raise NotImplementedError('projection units other than metres: %s' % proj4)
        self.proj4 = str(proj4)
        self.a = a
        self.lat_0, self.lon_0 = float(p.get('lat_0', 0.0)), float(p.get('lon_0', 0.0))
        self.has_lat_ts = 'lat_ts' in p
        self.lat_ts = float(p.get('lat_ts', 90.0))
        self.k_0 = float(p.get('k_0', p.get('k', 1.0)))
        self.x_0, self.y_0 = float(p.get('x_0', 0.0)), float(p.get('y_0', 0.0))
        phi0 = self.lat_0 * _DEG
        t = abs(phi0)
        if abs(t - np.pi / 2) < 1e-10:
            self.mode = 'S_POLE' if phi0 < 0 else 'N_POLE'
        else:
            self.mode = 'OBLIQ' if t > 1e-10 else 'EQUIT'
        self.phi0, self.lam0 = phi0, self.lon_0 * _DEG
        self.sinX1, self.cosX1 = np.sin(phi0), np.cos(phi0)
        phits = abs(self.lat_ts * _DEG) if self.has_lat_ts else np.pi / 2
        if self.mode in ('OBLIQ', 'EQUIT') or abs(phits - np.pi / 2) < 1e-10:
            self.akm1 = 2.0 * self.k_0
        else:
            self.akm1 = np.cos(phits) / np.tan(np.pi / 4 - 0.5 * phits)

    def desc(self):
        d = _lib.ProjDesc()
        d.kind = _lib.OD_PROJ_STERE_SPHERE
        d.has_lat_ts = 1 if self.has_lat_ts else 0
        d.a, d.lat_0, d.lon_0, d.lat_ts = self.a, self.lat_0, self.lon_0, self.lat_ts
        d.k_0, d.x_0, d.y_0 = self.k_0, self.x_0, self.y_0
        return d

    @staticmethod
    def _adjlon(lam):
        lam = np.asarray(lam, dtype=np.float64)
        return np.where(np.abs(lam) > np.pi, np.mod(lam + np.pi, 2 * np.pi) - np.pi, lam)

    def __call__(self, a, b, inverse=False):
        scalar = np.isscalar(a)
        a = np.atleast_1d(np.asarray(a, dtype=np.float64))
        b = np.atleast_1d(np.asarray(b, dtype=np.float64))
        ra, rb = self._inverse(a, b) if inverse else self._forward(a, b)
        if scalar:
            return float(ra[0]), float(rb[0])
        return ra, rb

    def _forward(self, lon, lat):
        lam = self._adjlon(lon * _DEG - self.lam0)
        phi = lat * _DEG
        sp, cp, sl, cl = np.sin(phi), np.cos(phi), np.sin(lam), np.cos(lam)
        with np.errstate(all='ignore'):
            if self.mode == 'EQUIT':
                k = self.akm1 / (1.0 + cp * cl)
                x, y = k * cp * sl, k * sp
            elif self.mode == 'OBLIQ':
                k = self.akm1 / (1.0 + self.sinX1 * sp + self.cosX1 * cp * cl)
                x, y = k * cp * sl, k * (self.cosX1 * sp - self.sinX1 * cp * cl)
            else:
                if self.mode == 'N_POLE':
                    cl, phi = -cl, -phi
                y = self.akm1 * np.tan(np.pi / 4 + 0.5 * phi)
                x, y = sl * y, y * cl
        return self.a * x + self.x_0, self.a * y + self.y_0

    def _inverse(self, x, y):
        x = (x - self.x_0) / self.a
        y = (y - self.y_0) / self.a
        rh = np.hypot(x, y)
        c = 2.0 * np.arctan(rh / self.akm1)
        sc, cc = np.sin(c), np.cos(c)
        small = rh <= 1e-10
        rhs = np.where(small, 1.0, rh)
        with np.errstate(all='ignore'):
            if self.mode == 'EQUIT':
                phi = np.where(small, 0.0, np.arcsin(np.clip(y * sc / rhs, -1, 1)))
                lam = np.where((cc != 0) | (x != 0), np.arctan2(x * sc, cc * rh), 0.0)
            elif self.mode == 'OBLIQ':
                phi = np.where(small, self.phi0, np.arcsin(np.clip(cc * self.sinX1 + y * sc * self.cosX1 / rhs, -1, 1)))
                d = cc - self.sinX1 * np.sin(phi)
                lam = np.where((d != 0) | (x != 0), np.arctan2(x * sc * self.cosX1, d * rh), 0.0)
            else:
                if self.mode == 'N_POLE':
                    y = -y
                phi = np.where(small, self.phi0, np.arcsin(-cc if self.mode == 'S_POLE' else cc))
                lam = np.where((x == 0) & (y == 0), 0.0, np.arctan2(x, y))
        return self._adjlon(lam + self.lam0) / _DEG, phi / _DEG


ELLIPSOIDS = {'WGS84': (6378137.0, 298.257223563), 'GRS80': (6378137.0, 298.257222101), 'sphere': (6370997.0, 0.0)}


def _ellipsoid(p, proj4):
    """(a, es) from +R / +a / +b / +rf / +f / +e / +es / +ellps / +datum=WGS84; an ellipsoid must be named."""
    if 'R' in p:
        return float(p['R']), 0.0
    a = rf = None
    if 'ellps' in p or p.get('datum') == 'WGS84':
        name = p.get('ellps', 'WGS84')
        if name not in ELLIPSOIDS:
            raise NotImplementedError('ellipsoid %s is not known to the GPU path: %s' % (name, proj4))
        a, rf = ELLIPSOIDS[name]
    if 'a' in p:
        a = float(p['a'])
    if a is None:
        raise NotImplementedError('the projection names no ellipsoid (+R, +a, +ellps, +datum=WGS84): %s' % proj4)
    if 'es' in p:
        es = float(p['es'])
    elif 'e' in p:
        es = float(p['e']) ** 2
    elif 'rf' in p:
        f = 1.0 / float(p['rf'])
        es = f * (2.0 - f)
    elif 'f' in p:
        f = float(p['f'])
        es = f * (2.0 - f)
    elif 'b' in p:
        es = 1.0 - (float(p['b']) / a) ** 2
    elif rf:
        f = 1.0 / rf
        es = f * (2.0 - f)
    else:
        es = 0.0
    return a, es


class _Conformal:
    """Mercator / Lambert conformal conic: parameters for od_proj_desc and the same closed forms in NumPy for the host points."""
    kind = None

    def __init__(self, proj4, name):
        p = parse_proj4(proj4)
        if p.get('proj') != name:
            raise NotImplementedError(proj4)
        if p.get('units', 'm') != 'm':
            raise NotImplementedError('projection units other than metres: %s' % proj4)
        self.proj4, self.p = str(proj4), p
        self.a, self.es = _ellipsoid(p, proj4)
        self.e = float(np.sqrt(self.es))
        self.lon_0 = float(p.get('lon_0', 0.0))
        self.lam0 = self.lon_0 * _DEG
        self.k_0 = float(p.get('k_0', p.get('k', 1.0)))
        self.x_0, self.y_0 = float(p.get('x_0', 0.0)), float(p.get('y_0', 0.0))
        self.lat_0 = float(p.get('lat_0', 0.0))
        self.has_lat_ts, self.lat_ts = False, 0.0
        self.lat_1 = self.lat_2 = 0.0

    def desc(self):
        d = _lib.ProjDesc()
        d.kind = self.kind
        d.has_lat_ts = 1 if self.has_lat_ts else 0
        d.a, d.lat_0, d.lon_0, d.lat_ts = self.a, self.lat_0, self.lon_0, self.lat_ts
        d.k_0, d.x_0, d.y_0 = self.k_0, self.x_0, self.y_0
        d.es, d.lat_1, d.lat_2 = self.es, self.lat_1, self.lat_2
        return d

    _adjlon = staticmethod(SphericalStereographic._adjlon)

    def _msfn(self, sinphi, cosphi):
        return cosphi / np.sqrt(1.0 - self.es * sinphi * sinphi)

    def _tsfn(self, phi):
        s = np.sin(phi)
        return np.tan(0.5 * (0.5 * np.pi - phi)) / np.power((1.0 - self.e * s) / (1.0 + self.e * s), 0.5 * self.e)

    def _phi2(self, ts):
        phi = 0.5 * np.pi - 2.0 * np.arctan(ts)
        for _ in range(20):
            con = self.e * np.sin(phi)
            new = 0.5 * np.pi - 2.0 * np.arctan(ts * np.power((1.0 - con) / (1.0 + con), 0.5 * self.e))
            d = np.max(np.abs(new - phi)) if np.size(new) else 0.0
            phi = new
            if d < 1e-14:
                break
        return phi

    def __call__(self, a, b, inverse=False):
        scalar = np.isscalar(a)
        a = np.atleast_1d(np.asarray(a, dtype=np.float64))
        b = np.atleast_1d(np.asarray(b, dtype=np.float64))
        with np.errstate(all='ignore'):
            if inverse:
                lam, phi = self._inv((a - self.x_0) / self.a, (b - self.y_0) / self.a)
                ra, rb = self._adjlon(lam + self.lam0) / _DEG, phi / _DEG
            else:
                x, y = self._fwd(self._adjlon(a * _DEG - self.lam0), b * _DEG)
                ra, rb = self.a * x + self.x_0, self.a * y + self.y_0
        if scalar:
            return float(ra[0]), float(rb[0])
        return ra, rb


class Mercator(_Conformal):
    kind = _lib.OD_PROJ_MERC

    def __init__(self, proj4):
        super().__init__(proj4, 'merc')
        self.kscale = self.k_0
        if 'lat_ts' in self.p:
            self.has_lat_ts, self.lat_ts = True, float(self.p['lat_ts'])
            phits = abs(self.lat_ts) * _DEG
            if phits >= 0.5 * np.pi:
                raise ValueError('+lat_ts must be below 90 degrees: %s' % proj4)
            self.kscale = float(self._msfn(np.sin(phits), np.cos(phits)))

    def _fwd(self, lam, phi):
        return self.kscale * lam, self.kscale * (np.arcsinh(np.tan(phi)) - self.e * np.arctanh(self.e * np.sin(phi)))

    def _inv(self, x, y):
        ts = np.exp(-y / self.kscale)
        return x / self.kscale, (self._phi2(ts) if self.es != 0.0 else 0.5 * np.pi - 2.0 * np.arctan(ts))


class LambertConformalConic(_Conformal):
    kind = _lib.OD_PROJ_LCC

    def __init__(self, proj4):
        super().__init__(proj4, 'lcc')
        p = self.p
        if 'lat_1' not in p:
            raise NotImplementedError('+proj=lcc needs +lat_1: %s' % proj4)
        self.lat_1 = float(p['lat_1'])
        self.lat_2 = float(p.get('lat_2', self.lat_1))
        self.lat_0 = float(p.get('lat_0', self.lat_1 if 'lat_2' not in p else 0.0))
        phi1, phi2, phi0 = self.lat_1 * _DEG, self.lat_2 * _DEG, self.lat_0 * _DEG
        if abs(phi1 + phi2) < 1e-10:
            raise ValueError('+lat_1 = -+lat_2: %s' % proj4)
        sinphi, cosphi = np.sin(phi1), np.cos(phi1)
        n = sinphi
        secant = abs(phi1 - phi2) >= 1e-10
        polar0 = abs(abs(phi0) - 0.5 * np.pi) < 1e-10
        if self.es != 0.0:
            m1, ml1 = self._msfn(sinphi, cosphi), self._tsfn(phi1)
            if secant:
                n = np.log(m1 / self._msfn(np.sin(phi2), np.cos(phi2))) / np.log(ml1 / self._tsfn(phi2))
            c = m1 * np.power(ml1, -n) / n
            rho0 = 0.0 if polar0 else c * np.power(self._tsfn(phi0), n)
        else:
            if secant:
                n = np.log(cosphi / np.cos(phi2)) / np.log(np.tan(0.25 * np.pi + 0.5 * phi2) / np.tan(0.25 * np.pi + 0.5 * phi1))
            c = cosphi * np.power(np.tan(0.25 * np.pi + 0.5 * phi1), n) / n
            rho0 = 0.0 if polar0 else c * np.power(np.tan(0.25 * np.pi + 0.5 * phi0), -n)
        self.n, self.c, self.rho0 = float(n), float(c), float(rho0)

    def _fwd(self, lam, phi):
        rho = self.c * (np.power(self._tsfn(phi), self.n) if self.es != 0.0 else np.power(np.tan(0.25 * np.pi + 0.5 * phi), -self.n))
        rho = np.where(np.abs(np.abs(phi) - 0.5 * np.pi) < 1e-10, np.where(phi * self.n > 0, 0.0, np.nan), rho)
        lam = lam * self.n
        return self.k_0 * rho * np.sin(lam), self.k_0 * (self.rho0 - rho * np.cos(lam))

    def _inv(self, x, y):
        x = x / self.k_0
        y = self.rho0 - y / self.k_0
        rho = np.hypot(x, y)
        if self.n < 0:
            rho, x, y = -rho, -x, -y
        safe = np.where(rho != 0, rho, 1.0)
        phi = self._phi2(np.power(safe / self.c, 1.0 / self.n)) if self.es != 0.0 \
            else 2.0 * np.arctan(np.power(self.c / safe, 1.0 / self.n)) - 0.5 * np.pi
        lam = np.arctan2(x, y) / self.n
        return np.where(rho != 0, lam, 0.0), np.where(rho != 0, phi, 0.5 * np.pi if self.n > 0 else -0.5 * np.pi)


class StereographicEllipsoid(_Conformal):
    """+proj=stere on an ellipsoid (Snyder eqs. 21-24 .. 21-40 through the conformal latitude; PROJ's stere.cpp, ellipsoidal half)."""
    kind = _lib.OD_PROJ_STERE_ELLPS

    def __init__(self, proj4):
        super().__init__(proj4, 'stere')
        p = self.p
        self.has_lat_ts = 'lat_ts' in p
        self.lat_ts = float(p.get('lat_ts', 90.0))
        phits = abs(self.lat_ts) * _DEG if self.has_lat_ts else 0.5 * np.pi
        phi0 = self.lat_0 * _DEG
        t = abs(phi0)
        if abs(t - 0.5 * np.pi) < 1e-10:
            self.mode = 'S_POLE' if phi0 < 0 else 'N_POLE'
        else:
            self.mode = 'OBLIQ' if t > 1e-10 else 'EQUIT'
        e = self.e
        if self.mode in ('N_POLE', 'S_POLE'):
            if abs(phits - 0.5 * np.pi) < 1e-10:
                self.akm1 = 2.0 * self.k_0 / np.sqrt(np.power(1 + e, 1 + e) * np.power(1 - e, 1 - e))
            else:
                self.akm1 = float(self._msfn(np.sin(phits), np.cos(phits)) / self._tsfn(phits))
            self.sinX1 = self.cosX1 = 0.0
        else:
            sp = np.sin(phi0)
            X = 2.0 * np.arctan(self._ssfn(phi0)) - 0.5 * np.pi
            self.akm1 = 2.0 * self.k_0 * np.cos(phi0) / np.sqrt(1.0 - self.es * sp * sp)
            self.sinX1, self.cosX1 = float(np.sin(X)), float(np.cos(X))

    def _ssfn(self, phi):
        s = self.e * np.sin(phi)
        return np.tan(0.5 * (0.5 * np.pi + phi)) * np.power((1.0 - s) / (1.0 + s), 0.5 * self.e)

    def _fwd(self, lam, phi):
        sl, cl = np.sin(lam), np.cos(lam)
        if self.mode in ('OBLIQ', 'EQUIT'):
            X = 2.0 * np.arctan(self._ssfn(phi)) - 0.5 * np.pi
            sX, cX = np.sin(X), np.cos(X)
            if self.mode == 'OBLIQ':
                A = self.akm1 / (self.cosX1 * (1.0 + self.sinX1 * sX + self.cosX1 * cX * cl))
                return A * cX * sl, A * (self.cosX1 * sX - self.sinX1 * cX * cl)
            A = self.akm1 / (1.0 + cX * cl)
            return A * cX * sl, A * sX
        if self.mode == 'S_POLE':
            phi, cl = -phi, -cl
        rho = self.akm1 * self._tsfn(phi)
        return rho * sl, -rho * cl

    def _inv(self, x, y):
        rho = np.hypot(x, y)
        e = self.e
        if self.mode in ('OBLIQ', 'EQUIT'):
            tp = 2.0 * np.arctan2(rho * self.cosX1, self.akm1)
            ct, st = np.cos(tp), np.sin(tp)
            safe = np.where(rho != 0, rho, 1.0)
            phi_l = np.where(rho == 0.0, np.arcsin(ct * self.sinX1), np.arcsin(np.clip(ct * self.sinX1 + y * st * self.cosX1 / safe, -1, 1)))
            tp = np.tan(0.5 * (0.5 * np.pi + phi_l))
            xx, yy = x * st, rho * self.cosX1 * ct - y * self.sinX1 * st
            halfpi, halfe = 0.5 * np.pi, 0.5 * e
        else:
            if self.mode == 'N_POLE':
                y = -y
            tp = -rho / self.akm1
            phi_l = 0.5 * np.pi - 2.0 * np.arctan(-tp)
            xx, yy = x, y
            halfpi, halfe = -0.5 * np.pi, -0.5 * e
        phi = phi_l
        for _ in range(20):
            sp = e * np.sin(phi_l)
            phi = 2.0 * np.arctan(tp * np.power((1.0 + sp) / (1.0 - sp), halfe)) - halfpi
            d = np.max(np.abs(phi_l - phi)) if np.size(phi) else 0.0
            phi_l = phi
            if d < 1e-14:
                break
        if self.mode == 'S_POLE':
            phi = -phi
        return np.where((xx == 0.0) & (yy == 0.0), 0.0, np.arctan2(xx, yy)), phi


def _is_sphere(proj4):
    p = parse_proj4(proj4)
    if 'R' in p:
        return True
    if any(k in p for k in ('ellps', 'datum', 'rf', 'f', 'b')):
        return _ellipsoid(p, proj4)[1] == 0.0
    es = float(p['e']) ** 2 if 'e' in p else float(p.get('es', 0.0))
    return es == 0.0


def is_rotated_pole(proj4):
    return parse_proj4(proj4).get('proj') == 'ob_tran'


class RotatedPole:
    """+proj=ob_tran +o_proj=longlat in its new-pole form (+o_lat_p, +o_lon_p, +lon_0; PROJ's ob_tran.cpp o_forward / o_inverse,
    Snyder 1987 eqs. 5-7 and 5-8b): the reader's plane is rotated longitude / latitude in DEGREES -- what the reference's lonlat2xy
    and xy2lonlat hand out around pyproj's radians (variables.py:111-143).  The rotation does not depend on the radius."""
    kind = _lib.OD_PROJ_OB_TRAN
    _REFUSED = ('to_meter', 'o_alpha', 'o_lon_c', 'o_lat_c', 'o_lon_1', 'o_lat_1', 'o_lon_2', 'o_lat_2', 'o_lon_b', 'o_lat_b')

    def __init__(self, proj4):
        p = parse_proj4(proj4)
        if p.get('proj') != 'ob_tran':
            raise NotImplementedError(proj4)
        if p.get('o_proj') not in ('longlat', 'lonlat', 'latlong'):
            raise NotImplementedError('+proj=ob_tran on the GPU path: +o_proj=longlat only; got %s' % proj4)
        bad = [k for k in self._REFUSED if k in p]
        if bad or 'o_lat_p' not in p:
            raise NotImplementedError('+proj=ob_tran on the GPU path: the +o_lat_p [+o_lon_p] form without +to_meter; got %s' % proj4)
        if any(float(p.get(k, 0.0)) != 0.0 for k in ('x_0', 'y_0')) or float(p.get('k_0', p.get('k', 1.0))) != 1.0:
            raise NotImplementedError('+proj=ob_tran with a false origin or a scale factor: %s' % proj4)
        self.proj4, self.p = str(proj4), p
        self.a = float(p['R']) if 'R' in p else float(p.get('a', 6378137.0))
        self.lon_0 = float(p.get('lon_0', 0.0))
        self.o_lat_p = float(p['o_lat_p'])
        self.o_lon_p = float(p.get('o_lon_p', 0.0))
        if not (abs(self.o_lat_p) <= 90.0):
            raise ValueError('+o_lat_p must lie in [-90, 90]: %s' % proj4)
        self.lam0, self.lamp = self.lon_0 * _DEG, self.o_lon_p * _DEG
        self.sphip, self.cphip = np.sin(self.o_lat_p * _DEG), np.cos(self.o_lat_p * _DEG)

    def desc(self):
        d = _lib.ProjDesc()
        d.kind = self.kind
        d.a, d.lon_0, d.k_0 = self.a, self.lon_0, 1.0
        d.lat_1, d.lat_2 = self.o_lat_p, self.o_lon_p
        return d

    _adjlon = staticmethod(SphericalStereographic._adjlon)

    def __call__(self, a, b, inverse=False):
        scalar = np.isscalar(a)
        a = np.atleast_1d(np.asarray(a, dtype=np.float64))
        b = np.atleast_1d(np.asarray(b, dtype=np.float64))
        with np.errstate(all='ignore'):
            if inverse:
                lam, phi = np.radians(a) - self.lamp, np.radians(b)
                sl, cl, sp, cp = np.sin(lam), np.cos(lam), np.sin(phi), np.cos(phi)
                ra = np.degrees(self._adjlon(np.arctan2(cp * sl, self.sphip * cp * cl - self.cphip * sp) + self.lam0))
                rb = np.degrees(np.arcsin(np.clip(self.sphip * sp + self.cphip * cp * cl, -1, 1)))
            else:
                lam, phi = self._adjlon(a * _DEG - self.lam0), b * _DEG
                sl, cl, sp, cp = np.sin(lam), np.cos(lam), np.sin(phi), np.cos(phi)
                ra = np.degrees(self._adjlon(np.arctan2(cp * sl, self.sphip * cp * cl + self.cphip * sp) + self.lamp))
                rb = np.degrees(np.arcsin(np.clip(self.sphip * sp - self.cphip * cp * cl, -1, 1)))
        if scalar:
            return float(ra[0]), float(rb[0])
        return ra, rb


def make_projection(proj4):
    """The projection object of a reader's proj4 string (None for a geographic reader)."""
    if is_rotated_pole(proj4):                 # (before the geographic test: its +o_proj=longlat names a geographic CRS)
        return RotatedPole(proj4)
    if is_geographic(proj4):
        return None
    name = parse_proj4(proj4).get('proj')
    if name == 'stere':
        return SphericalStereographic(proj4) if _is_sphere(proj4) else StereographicEllipsoid(proj4)
    if name == 'merc':
        return Mercator(proj4)
    if name == 'lcc':
        return LambertConformalConic(proj4)
    raise NotImplementedError('projected readers on the GPU path: +proj=stere, +proj=merc, +proj=lcc; got %s' % proj4)
