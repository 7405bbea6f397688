"""ORACLE (test infrastructure, never the product path).

CPU restatement, in NumPy float64, of the rotated pole '+proj=ob_tran +o_proj=longlat +o_lat_p=.. [+o_lon_p=..] +lon_0=..', the grid
mapping of CF 'rotated_latitude_longitude' forcing (reader_netCDF_CF_generic.py:145-161 turns it into this proj4 string), and
``install()``, which adds it to the fake ``pyproj`` of oracle/refrun.py (after ``refrun.setup()``, before any reader is built).

The rotation is the spherical oblique transformation of J. P. Snyder, "Map Projections: A Working Manual" (USGS PP 1395, 1987),
eqs. 5-7 and 5-8b, organised the way PROJ's ob_tran.cpp organises it (o_forward / o_inverse): lam = lon - lon_0 reduced to
[-pi, pi]; the pole moves to latitude o_lat_p; o_lon_p is added to the rotated longitude, which is reduced to [-pi, pi] again.
It does not depend on the radius.

Units -- pyproj's documented conventions for an ob_tran CRS whose o_proj is longlat, which the reference's code is written
around (variables.py:111-143 applies np.degrees / np.radians around Proj calls):
  * ``Proj(lon, lat)`` takes degrees and returns the rotated coordinates in RADIANS; ``Proj(x, y, inverse=True)`` takes
    radians and returns degrees;
  * ``crs.is_geographic`` is True;
  * a ``Transformer`` from such a CRS takes rotated DEGREES.

Pinning: PARITY UNPINNED against a PROJ binary -- neither pyproj nor PROJ is available where the fixtures are written, so these
conventions are taken from pyproj's documentation and cannot be checked against it here.  tests/test_rotpole_host.py checks the
rotation against the closed forms evaluated independently with mpmath at 40 digits, the two known answers (rotated (0, 0) is
true (lon_0, 90 - o_lat_p); true (lon_0 + 180, o_lat_p) has rotated latitude 90), and round trips.
"""
import numpy as np

from oracle.proj_stere import parse_proj4

_DEG = np.pi / 180.0


def _adjlon(lam):
    lam = np.asarray(lam, dtype=np.float64)
    return np.where(np.abs(lam) > np.pi, np.mod(lam + np.pi, 2 * np.pi) - np.pi, lam)


def is_ob_tran(proj4):
    return parse_proj4(proj4).get('proj') == 'ob_tran'


class ObTran:
    def __init__(self, proj4):
        p = parse_proj4(proj4)
        if p.get('proj') != 'ob_tran' or p.get('o_proj') not in ('longlat', 'lonlat', 'latlong') or 'o_lat_p' not in p:
            raise NotImplementedError('fake pyproj: ob_tran with +o_proj=longlat and +o_lat_p only: ' + str(proj4))
        self.p = p
        self.lon_0 = float(p.get('lon_0', 0.0))
        self.o_lat_p = float(p['o_lat_p'])
        self.o_lon_p = float(p.get('o_lon_p', 0.0))
        self.lam0, self.lamp = self.lon_0 * _DEG, self.o_lon_p * _DEG
        self.sphip, self.cphip = np.sin(self.o_lat_p * _DEG), np.cos(self.o_lat_p * _DEG)

    def forward(self, lon, lat):
        """degrees -> rotated radians (what pyproj's Proj returns)"""
        lam = _adjlon(np.asarray(lon, dtype=np.float64) * _DEG - self.lam0)
        phi = np.asarray(lat, dtype=np.float64) * _DEG
        sl, cl, sp, cp = np.sin(lam), np.cos(lam), np.sin(phi), np.cos(phi)
        x = _adjlon(np.arctan2(cp * sl, self.sphip * cp * cl + self.cphip * sp) + self.lamp)
        y = np.arcsin(np.clip(self.sphip * sp - self.cphip * cp * cl, -1.0, 1.0))
        return x, y

    def inverse(self, x, y):
        """rotated radians -> degrees"""
        lam = np.asarray(x, dtype=np.float64) - self.lamp
        phi = np.asarray(y, dtype=np.float64)
        sl, cl, sp, cp = np.sin(lam), np.cos(lam), np.sin(phi), np.cos(phi)
        lat = np.arcsin(np.clip(self.sphip * sp + self.cphip * cp * cl, -1.0, 1.0))
        lon = _adjlon(np.arctan2(cp * sl, self.sphip * cp * cl - self.cphip * sp) + self.lam0)
        return np.degrees(lon), np.degrees(lat)

    def forward_deg(self, lon, lat):
        """degrees -> rotated degrees (the reference's lonlat2xy)"""
        x, y = self.forward(lon, lat)
        return np.degrees(x), np.degrees(y)

    def inverse_deg(self, x, y):
        """rotated degrees -> degrees (the reference's xy2lonlat, and a Transformer from the ob_tran CRS)"""
        return self.inverse(np.radians(np.asarray(x, dtype=np.float64)), np.radians(np.asarray(y, dtype=np.float64)))


def install():
    """Extend the fake ``pyproj`` module that oracle/refrun.py installs with the ob_tran stand-in: ``Proj`` and ``Transformer``
    become subclasses that serve ob_tran CRSs and hand everything else to the classes they extend.  The reference compares
    ``type(proj) is pyproj.Proj`` (variables.py:73-77), so this must run before any reader is built.  Idempotent."""
    import sys
    pyproj = sys.modules['pyproj']
    if getattr(pyproj, 'ob_tran_installed', False):
        return
    BaseProj, BaseTransformer = pyproj.Proj, pyproj.Transformer
    CRS = type(BaseProj('+proj=latlong').crs)

    class Proj(BaseProj):
        """ob_tran: geographic to pyproj; degrees in and radians out forward, radians in and degrees out inverse"""

        def __init__(self, projparams=None, **kw):
            s = str(projparams)
            if not is_ob_tran(s):
                super().__init__(projparams, **kw)
                return
            self.srs = s
            self.definition_string = lambda: s
            self.impl = ObTran(s)
            self.crs = CRS(True, s)

    class Transformer(BaseTransformer):
        @classmethod
        def from_proj(cls, proj_from, proj_to, **kw):
            pf = proj_from if isinstance(proj_from, BaseProj) else Proj(proj_from)
            pt = proj_to if isinstance(proj_to, BaseProj) else Proj(proj_to)
            return cls(pf, pt)

        def transform(self, x, y):
            if not is_ob_tran(self.pf.srs):
                return super().transform(x, y)
            scalar = np.isscalar(x)                     # a Transformer takes the rotated coordinates in degrees
            lon, lat = self.pf.impl.inverse_deg(x, y)
            if scalar:
                lon, lat = float(lon), float(lat)
            return self.pt(lon, lat)

    pyproj.Proj, pyproj.Transformer = Proj, Transformer
    pyproj.ob_tran_installed = True
