"""Gridded readers on a rotated-pole grid (+proj=ob_tran +o_proj=longlat, tests/rotpolecases.py) on the host build of the device
sources: the oracle's rotation against the closed forms at 40 digits, the device rotation against the oracle, the reader's host
helpers and refusals, and the drop-in model classes against runs of the unmodified reference."""
import ctypes as C

import numpy as np
import pytest

import common
import rotpolecases as rc
from hostengine import HostEngine

PROJS = [rc.WAM, rc.ROT_EAST, rc.CROSS_EAST,
         '+proj=ob_tran +o_proj=longlat +o_lon_p=-30 +o_lat_p=-40 +lon_0=150 +R=6371000 +no_defs',
         '+proj=ob_tran +o_proj=lonlat +o_lat_p=0 +lon_0=0 +R=6371000 +no_defs']


@pytest.fixture()
def host_engine(monkeypatch):
    eng = HostEngine()
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    monkeypatch.setattr(E, 'default_engine', lambda device=None: eng)
    monkeypatch.setattr(B, 'default_engine', lambda device=None: eng)
    yield eng


def _random(P, n, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(-180, 180, n), np.degrees(np.arcsin(rng.uniform(-0.999, 0.999, n)))


@pytest.mark.parametrize('proj4', PROJS)
def test_rotated_pole_oracle_against_mpmath(proj4):
    """Snyder 5-7 / 5-8b written independently: the rotated pole is the true point (lon_0 + 180, o_lat_p); rotated latitude =
    asin(sin phi sin phi_p + cos phi cos phi_p cos(lam - lam_p)) with lam_p = lon_0 + 180, rotated longitude measured from the
    meridian through the true pole, plus o_lon_p."""
    import mpmath as mp
    from oracle.proj_obtran import ObTran
    mp.mp.dps = 40
    P = ObTran(proj4)
    lon, lat = _random(P, 60, 5)
    x, y = P.forward(lon, lat)
    php, lamp = mp.radians(mp.mpf(P.o_lat_p)), mp.radians(mp.mpf(P.lon_0) + 180)
    for i in range(len(lon)):
        phi, lam = mp.radians(mp.mpf(float(lat[i]))), mp.radians(mp.mpf(float(lon[i])))
        ey = mp.asin(mp.sin(phi) * mp.sin(php) + mp.cos(phi) * mp.cos(php) * mp.cos(lam - lamp))
        ex = mp.atan2(mp.cos(phi) * mp.sin(lam - lamp), mp.sin(php) * mp.cos(phi) * mp.cos(lam - lamp) - mp.cos(php) * mp.sin(phi))
        ex = ex + mp.pi + mp.radians(mp.mpf(P.o_lon_p))                     # measured from the meridian opposite the rotated pole's
        ex = ex - 2 * mp.pi * mp.floor((ex + mp.pi) / (2 * mp.pi))
        assert abs(float(ey) - y[i]) < 1e-14, (i, float(ey), y[i])
        d = float(ex) - x[i]
        assert abs(d - 2 * np.pi * round(d / (2 * np.pi))) < 1e-13, (i, float(ex), x[i])
    lo, la = P.inverse(x, y)
    assert np.max(np.abs((lo - lon + 180) % 360 - 180)) < 1e-9 and np.max(np.abs(la - lat)) < 1e-9
    # the known answers: rotated (0, 0) is true (lon_0, 90 - o_lat_p); true (lon_0 + 180, o_lat_p) is the rotated pole
    if P.o_lon_p == 0:
        lo, la = P.inverse(np.array([0.0]), np.array([0.0]))
        assert abs((lo[0] - P.lon_0 + 180) % 360 - 180) < 1e-12 and abs(la[0] - (90 - P.o_lat_p)) < 1e-12
    _, yp = P.forward(np.array([P.lon_0 + 180]), np.array([P.o_lat_p]))
    assert abs(np.degrees(yp[0]) - 90) < 1e-6


def test_fake_pyproj_serves_ob_tran_in_pyproj_units(monkeypatch):
    """oracle/proj_obtran.install() on the reference's fake pyproj: geographic CRS, radians out of Proj forward, radians into
    Proj inverse, degrees into a Transformer; other CRSs are served as before."""
    import sys
    from oracle import refrun
    from oracle.proj_obtran import ObTran, install
    if not refrun.available():
        pytest.skip('the reference is not installed')
    refrun.setup()
    pyproj = sys.modules['pyproj']
    for k in ('Proj', 'Transformer'):                                # (restored after the test)
        monkeypatch.setattr(pyproj, k, getattr(pyproj, k))
    monkeypatch.setattr(pyproj, 'ob_tran_installed', False, raising=False)
    install()
    O = ObTran(rc.WAM)
    p = pyproj.Proj(rc.WAM)
    assert p.crs.is_geographic and 'ob_tran' in p.srs and type(p) is pyproj.Proj
    lon, lat = np.array([3.0, 10.0]), np.array([58.0, 65.0])
    x, y = p(lon, lat)
    ex, ey = O.forward(lon, lat)
    assert np.array_equal(x, ex) and np.array_equal(y, ey) and np.max(np.abs(x)) < np.pi
    lo, la = p(x, y, inverse=True)
    assert np.max(np.abs(lo - lon)) < 1e-12 and np.max(np.abs(la - lat)) < 1e-12
    t = pyproj.Transformer.from_proj(p, '+proj=latlong')
    lo, la = t.transform(np.degrees(x), np.degrees(y))
    assert np.max(np.abs(lo - lon)) < 1e-12 and np.max(np.abs(la - lat)) < 1e-12
    assert pyproj.Proj('+proj=latlong')(3.0, 58.0) == (3.0, 58.0)


@pytest.mark.parametrize('proj4', PROJS)
def test_device_rotation_equals_the_oracle(proj4):
    from opendrift_b200.readers.projection import make_projection
    from oracle.proj_obtran import ObTran
    lib = common.hostshim()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)                   # noqa: E731
    P, O = make_projection(proj4), ObTran(proj4)
    n = 20000
    lon, lat = _random(O, n, 1)
    ox, oy = O.forward_deg(lon, lat)
    px, py = P(lon, lat)
    assert np.array_equal(px, ox) and np.array_equal(py, oy)      # the product's host-side rotation (seeding helper)
    d = P.desc()
    hx, hy, hl, ha = (np.empty(n) for _ in range(4))
    assert lib.hs_proj(C.byref(d), 0, C.c_int64(n), vp(lon), vp(lat), vp(hx), vp(hy)) == 0
    assert lib.hs_proj(C.byref(d), 1, C.c_int64(n), vp(ox), vp(oy), vp(hl), vp(ha)) == 0
    ol, oa = O.inverse_deg(ox, oy)
    dx = (hx - ox + 180) % 360 - 180
    assert max(np.max(np.abs(dx)), np.max(np.abs(hy - oy))) <= 1e-12                       # rotated degrees
    assert max(np.max(np.abs((hl - ol + 180) % 360 - 180)), np.max(np.abs(ha - oa))) <= 1e-12
    ok = np.abs(lat) < 89.9                                        # (longitude is ill-conditioned at the true poles)
    assert np.max(np.abs(ha - lat)) < 1e-9 and np.max(np.abs(((hl - lon + 180) % 360 - 180)[ok])) < 1e-9


def test_rotated_pole_is_not_geographic():
    from opendrift_b200 import _lib
    from opendrift_b200.readers.projection import is_geographic, make_projection, RotatedPole
    s = '+proj=ob_tran +o_proj=longlat +o_lon_p=0 +o_lat_p=22 +lon_0=-40 +R=6370997 +no_defs'
    assert not is_geographic(s) and isinstance(make_projection(s), RotatedPole)
    assert is_geographic('+proj=longlat +ellps=WGS84') and make_projection('+proj=latlong') is None
    d = make_projection(s).desc()
    assert (d.kind, d.lon_0, d.lat_1, d.lat_2, d.a) == (_lib.OD_PROJ_OB_TRAN, -40.0, 22.0, 0.0, 6370997.0) and _lib.OD_PROJ_OB_TRAN == 5


def _reader(proj4, xs, ys, **kw):
    from opendrift_b200.readers import reader_regular_grid
    f = np.zeros((1, len(ys), len(xs)), dtype=np.float32)
    return reader_regular_grid.Reader(np.asarray(xs), np.asarray(ys), None, common.syn.slab_times(1),
                                      {common.CUR[0]: f, common.CUR[1]: f}, proj4=proj4, **kw)


def test_reader_host_helpers():
    r = _reader(rc.WAM, np.arange(-2, 2.01, 0.1), np.arange(-1, 1.01, 0.1))
    lo, la = r.xy2lonlat(0.0, 0.0)
    assert abs(lo - -40.0) < 1e-12 and abs(la - 68.0) < 1e-12
    x, y = r.lonlat2xy(lo, la)
    assert abs(x) < 1e-9 and abs(y) < 1e-9
    assert r.pixel_size() == r.delta_x * 111000                   # rotated degrees -> metres, as for a geographic reader
    assert not r.global_coverage()


def test_covers_positions_follows_the_true_corner_longitudes():
    """The rotated x is modulated with the convention of the TRUE corner longitudes before the box test: on a grid whose true
    corners all lie east of Greenwich, an element west of rotated x = 0 is tested as x + 360 and is not covered."""
    from oracle.proj_obtran import ObTran
    r = _reader(rc.ROT_EAST, np.arange(-0.86, 0.87, 0.04), np.arange(-0.74, 0.75, 0.04))
    O = ObTran(rc.ROT_EAST)
    lon, lat = O.inverse_deg(np.array([-0.5, 0.5, 0.0]), np.array([0.1, 0.1, 0.0]))
    ind, x, y = r.covers_positions(lon, lat)
    assert list(ind) == [1, 2]
    assert abs(x[0] - 0.5) < 1e-9                                 # (the unmodulated rotated x is handed back)


@pytest.mark.parametrize('proj4, err', [
    ('+proj=ob_tran +o_proj=merc +o_lat_p=30 +lon_0=0 +R=6371000', NotImplementedError),
    ('+proj=ob_tran +o_proj=longlat +o_lat_p=30 +lon_0=0 +to_meter=0.0174532925199 +R=6371000', NotImplementedError),
    ('+proj=ob_tran +o_proj=longlat +o_lat_p=30 +o_alpha=20 +lon_0=0 +R=6371000', NotImplementedError),
    ('+proj=ob_tran +o_proj=longlat +o_lon_c=10 +o_lat_c=50 +o_alpha=0 +R=6371000', NotImplementedError),
    ('+proj=ob_tran +o_proj=longlat +o_lon_1=10 +o_lat_1=50 +o_lon_2=30 +o_lat_2=40 +R=6371000', NotImplementedError),
    ('+proj=ob_tran +o_proj=longlat +lon_0=0 +R=6371000', NotImplementedError),
])
def test_unsupported_rotated_pole_forms_are_refused(proj4, err):
    from opendrift_b200.readers.projection import make_projection
    with pytest.raises(err):
        make_projection(proj4)


def test_unsupported_rotated_grids_are_refused():
    with pytest.raises(NotImplementedError):                      # 360 degrees of rotated longitude
        _reader(rc.WAM, np.arange(-180, 180, 1.0), np.arange(-10, 10.1, 1.0))
    with pytest.raises(NotImplementedError):
        _reader(rc.WAM, np.arange(0, 360, 1.0), np.arange(-10, 10.1, 1.0))
    with pytest.raises(NotImplementedError):                      # the y-axis line would cross the rotated pole
        _reader(rc.WAM, np.arange(-10, 10.1, 1.0), np.arange(70, 89.95, 0.1))
    with pytest.raises(NotImplementedError):
        _reader(rc.WAM, np.arange(-10, 10.1, 1.0), np.arange(-90, -80, 1.0))
    with pytest.raises(NotImplementedError):                      # sub-block readers on a projected plane
        _reader(rc.WAM, np.arange(-10, 10.1, 1.0), np.arange(-10, 10.1, 1.0), subblocks=True)
    _reader(rc.WAM, np.arange(-10, 10.1, 1.0), np.arange(70, 89.8, 0.1))


@pytest.mark.parametrize('case', list(rc.CASES))
def test_rotated_pole_case_equals_the_reference(case, host_engine):
    o = rc.run_product(case)
    e, dz, moved = rc.check(o, case)
    assert moved > 5e-3
    assert e < 5e-8 and dz <= (1e-9 if 'mixing' in case else 1e-5), (e, dz)
    ref = np.load(rc.GOLDEN)
    lon0, lat0 = rc.setup(case)[6:8]
    assert rc.unmoved(o.elements.lon, o.elements.lat, lon0, lat0) == int(ref['%s__unmoved' % case])
