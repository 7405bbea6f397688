"""PlastDrift: cases shared by the CPU (host engine) and GPU tests.  The expected results come from the UNMODIFIED reference's
PlastDrift: tests/golden/plast_ref.npz, written by `python tests/plastcases.py` (oracle/refrun.py).  Every run records, after each
update(), the IDs, positions and depths of the active elements and whether the depths are float64; the end state includes the
deactivated elements in the order they were removed, with their status."""
import os
from datetime import datetime, timedelta

import numpy as np

import common

GOLDEN = os.path.join(common.GOLDEN, 'plast_ref.npz')
N, STEPS = 240, 8

_BASE = {'general:use_auto_landmask': False, 'seed:ocean_only': False, 'environment:constant:land_binary_mask': 0,
         'general:coastline_action': 'none'}
_RW = {'vertical_mixing:mixingmodel': 'randomwalk'}
_MASK = {'environment:constant:land_binary_mask': None, 'general:coastline_action': 'previous',
         'general:coastline_approximation_precision': None}
# name -> (config, readers among 'cur' / 'wind' / 'stokes' / 'hs' / 'k3d' / 'mld' / 'floor' / 'mask', seeding ('surface': the default
#          depth, a scalar; 'depth': float32 depths of 0 .. 40 m), terminal velocity (None: the default, a scalar), release over time,
#          time step in seconds (negative: backward))
CASES = {
    'analytical_tabularised': ({}, ('cur', 'wind'), 'surface', None, False, 900),
    'stokes_hs_readers': ({}, ('cur', 'wind', 'stokes', 'hs'), 'surface', None, False, 900),
    'monochromatic': ({'drift:stokes_drift_profile': 'monochromatic'}, ('cur', 'wind', 'stokes'), 'depth', None, False, 900),
    'exponential': ({'drift:stokes_drift_profile': 'exponential'}, ('cur', 'wind', 'stokes', 'hs'), 'depth', None, False, 900),
    'phillips': ({'drift:stokes_drift_profile': 'Phillips', 'drift:wind_drift_depth': 0}, ('cur', 'wind', 'stokes'), 'surface', None,
                 False, 900),
    'k_profile': ({}, ('cur', 'wind', 'k3d'), 'depth', None, False, 900),
    'mixed_terminal_velocity': ({'drift:wind_drift_depth': 2.0}, ('cur', 'wind', 'k3d'), 'depth', 'mixed', False, 900),
    'randomwalk_sundby_mld': (_RW, ('cur', 'wind', 'mld'), 'depth', None, False, 900),
    'randomwalk_environment': (dict(_RW, **{'vertical_mixing:diffusivitymodel': 'environment'}), ('cur', 'wind', 'k3d'), 'depth',
                               'mixed', False, 900),
    'no_mixing': ({'drift:vertical_mixing': False}, ('cur', 'wind', 'stokes'), 'depth', None, False, 900),
    'shallow_floor': ({}, ('cur', 'wind', 'floor'), 'surface', None, False, 900),
    'mask_previous': (_MASK, ('cur', 'wind', 'mask'), 'surface', None, True, 900),
    'release_backward': ({}, ('cur', 'wind', 'stokes'), 'depth', 'mixed', True, -900),
    'uncertainty': ({'drift:current_uncertainty': 0.1, 'drift:wind_uncertainty': 1.0}, ('cur', 'wind'), 'surface', None, True, 900),
    'subclass_reference_update': ({}, ('cur', 'wind', 'stokes', 'hs'), 'depth', 'mixed', False, 900),
}
# cases whose depths come from the random-walk mixing loop with a diffusivity from a non-zero wind (Sundby 1983): the wind speed of the
# analytical models differs from the reference's by an ulp here and there, which moves depths by about 1e-6 m
WIND_K = ('randomwalk_sundby_mld',)
RANDOMWALK = ('randomwalk_sundby_mld', 'randomwalk_environment')


def fields(fx):
    """float32 fields [nt, ny, nx] on the current grid: Stokes drift towards the north-east, Hs of 0.5 .. 4.5 m, a mixed layer of
    10 .. 40 m, a shallow sea floor of 3 .. 12 m, land in the easternmost columns."""
    X, Y = np.meshgrid(fx.grid_lon, fx.grid_lat)
    xs = (X - fx.grid_lon[0]) / (fx.grid_lon[-1] - fx.grid_lon[0])
    nt = len(fx.times)
    sx = np.stack([0.05 + 0.1 * xs + 0.01 * k for k in range(nt)]).astype(np.float32)
    sy = np.stack([0.12 - 0.05 * np.sin(4.0 * Y) + 0.0 * k for k in range(nt)]).astype(np.float32)
    hs = np.stack([2.5 + 2.0 * np.sin(3.0 * X + 0.5 * k) * np.cos(5.0 * Y) for k in range(nt)]).astype(np.float32)
    mld = np.stack([25.0 + 15.0 * np.sin(2.0 * X + 0.3 * k) * np.cos(3.0 * Y) for k in range(nt)]).astype(np.float32)
    floor = np.repeat((7.5 + 4.5 * np.sin(5.0 * X) * np.cos(4.0 * Y)).astype(np.float32)[None], nt, axis=0)
    mask = np.zeros(X.shape, dtype=np.float32)
    mask[:, fx.grid_lon > 3.6] = 1.0
    return sx, sy, hs, mld, floor, np.repeat(mask[None], nt, axis=0)


def terminal_velocity(kind, n):
    """None (the element default, a scalar), or float32 velocities of 0.002 .. 0.05 m/s."""
    if kind is None:
        return {}
    k = np.arange(n)
    return {'terminal_velocity': (0.002 + 0.048 * ((k * 7) % 17) / 16.0).astype(np.float32)}


def run_case(case, Model, make_reader, extra_config=None, ref_update=None, n=N, **model_kw):
    """The same script on the reference's classes and on the product's.  ref_update: the reference's PlastDrift.update, run by a
    subclass of Model (case 'subclass_reference_update')."""
    cfg, readers, seeding, tv, release, dt = CASES[case]
    cfg = dict(cfg, **(extra_config or {}))
    fx = common.Fixture('rk4_3d_full')
    sx, sy, hs, mld, floor, mask = fields(fx)

    class Recorder(Model):
        def update(self):
            if ref_update is not None:
                ref_update(self)
            else:
                super().update()
            el = self.elements
            z = np.atleast_1d(el.z)
            self.rec.append((np.array(el.ID, dtype=np.int64), np.array(el.lon, dtype=np.float64), np.array(el.lat, dtype=np.float64),
                             np.array(z, dtype=np.float64), z.dtype == np.float64))

    np.random.seed(11)
    o = Recorder(loglevel=50, **model_kw)
    o.rec = []
    grid2d = lambda f, name: make_reader(fx.grid_lon, fx.grid_lat, None, fx.times, f, name)       # noqa: E731
    comps = {}
    if 'cur' in readers:
        comps = {common.CUR[0]: fx.u, common.CUR[1]: fx.v}
    if 'k3d' in readers:
        comps['ocean_vertical_diffusivity'] = common.Fixture('rk4_3d_mixing').kdiff
    if comps:
        o.add_reader(make_reader(fx.grid_lon, fx.grid_lat, fx.grid_z, fx.times, comps, 'current'))
    if 'wind' in readers:
        o.add_reader(make_reader(fx.wind_lon, fx.wind_lat, None, fx.times, {'x_wind': fx.x_wind, 'y_wind': fx.y_wind}, 'wind'))
    comps = {}
    if 'stokes' in readers:
        comps['sea_surface_wave_stokes_drift_x_velocity'] = sx
        comps['sea_surface_wave_stokes_drift_y_velocity'] = sy
    if 'hs' in readers:
        comps['sea_surface_wave_significant_height'] = hs
    if 'mld' in readers:
        comps['ocean_mixed_layer_thickness'] = mld
    if 'floor' in readers:
        comps['sea_floor_depth_below_sea_level'] = floor
    if comps:
        o.add_reader(grid2d(comps, 'waves'))
    if 'mask' in readers:
        o.add_reader(grid2d({'land_binary_mask': mask}, 'mask'))
    config = dict(_BASE)
    config.update(cfg)
    for k, val in config.items():
        o.set_config(k, val)
    t0 = fx.start if dt > 0 else fx.times[-1]
    t = [t0, t0 + timedelta(seconds=3 * dt)] if release else t0
    kw = terminal_velocity(tv, n)
    if seeding == 'depth':
        kw['z'] = np.resize(np.maximum(fx.z0, np.float32(-40.0)), n).astype(np.float32)
    o.seed_elements(lon=np.resize(fx.lon0, n), lat=np.resize(fx.lat0, n), time=t, number=n, **kw)
    o.run(steps=STEPS, time_step=dt, time_step_output=dt)
    return o


def run_product(case, extra_config=None, n=N, **model_kw):
    from opendrift_b200.models.plastdrift import PlastDrift
    from opendrift_b200.readers import reader_regular_grid
    ref_update = None
    if case == 'subclass_reference_update':
        from oracle import refrun
        refrun.setup()
        from opendrift.models.plastdrift import PlastDrift as RefPlast
        ref_update = RefPlast.update
    return run_case(case, PlastDrift, lambda lon, lat, z, t, f, name: reader_regular_grid.Reader(lon, lat, z, t, f, name=name),
                    extra_config, ref_update=ref_update, n=n, **model_kw)


def run_shear(Model):
    """The reference's known answer (tests/models/test_models.py::test_wind_drift_shear) without the GSHHG landmask: three elements at
    0, 5 and 10 cm in a 10 m/s wind for ten hours.  Returns the final longitudes and latitudes."""
    o = Model(loglevel=50)
    o.set_config('general:use_auto_landmask', False)
    o.set_config('environment:fallback:x_wind', 10)
    o.set_config('environment:fallback:y_wind', 0)
    o.set_config('environment:fallback:land_binary_mask', 0)
    o.seed_elements(lat=60, lon=5, time=datetime(2024, 1, 1), number=3, z=np.array([0, -0.05, -.1]))
    o.run(duration=timedelta(hours=10))
    return np.asarray(o.elements.lon, dtype=np.float64), np.asarray(o.elements.lat, dtype=np.float64)


SHEAR_LON = [5.010873, 5.016866, 5.009735]


def summary(o):
    el, de = o.elements, o.elements_deactivated
    out = {'id': np.asarray(el.ID, dtype=np.int64), 'lon': np.asarray(el.lon, dtype=np.float64), 'lat': np.asarray(el.lat, dtype=np.float64),
           'z': np.asarray(el.z, dtype=np.float64), 'status': np.asarray(el.status, dtype=np.int64),
           'cats': np.array(list(o.status_categories))}
    if o.num_elements_deactivated():
        out.update({'d_id': np.asarray(de.ID, dtype=np.int64), 'd_lon': np.asarray(de.lon, dtype=np.float64),
                    'd_lat': np.asarray(de.lat, dtype=np.float64), 'd_z': np.asarray(de.z, dtype=np.float64),
                    'd_status': np.asarray(de.status, dtype=np.int64)})
    else:
        out.update({'d_id': np.zeros(0, np.int64), 'd_lon': np.zeros(0), 'd_lat': np.zeros(0), 'd_z': np.zeros(0),
                    'd_status': np.zeros(0, np.int64)})
    rec = o.rec
    out['h_len'] = np.array([len(r[0]) for r in rec], dtype=np.int64)
    out['h_id'] = np.concatenate([r[0] for r in rec]) if rec else np.zeros(0, np.int64)
    out['h_lon'] = np.concatenate([r[1] for r in rec]) if rec else np.zeros(0)
    out['h_lat'] = np.concatenate([r[2] for r in rec]) if rec else np.zeros(0)
    out['h_z'] = np.concatenate([r[3] for r in rec]) if rec else np.zeros(0)
    out['h_zf64'] = np.array([r[4] for r in rec], dtype=bool)
    return out


TOL_DEG = 5e-8


def _zdiff(a, b):
    """max |a - b| where both are finite; NaN and infinite depths must sit at the same places with the same values"""
    assert np.array_equal(np.isfinite(a), np.isfinite(b))
    assert np.array_equal(a[~np.isfinite(a)], b[~np.isfinite(b)], equal_nan=True)
    f = np.isfinite(a)
    return float(np.max(np.abs(a[f] - b[f]))) if f.any() else 0.0


def check(o, case, exact_z=True):
    """Returns (largest position difference in degrees, largest depth difference in m) against the reference.  exact_z: the
    analytical depths are the reference's bit for bit (legacy generator draws)."""
    ref = np.load(GOLDEN)
    got = summary(o)
    g = lambda k: ref['%s__%s' % (case, k)]                      # noqa: E731
    assert list(got['cats']) == list(g('cats')), (list(got['cats']), list(g('cats')))
    for k in ('id', 'status', 'd_id', 'd_status', 'h_len', 'h_id', 'h_zf64'):
        assert np.array_equal(got[k], g(k)), k
    # 'previous': an element moved back lands on the float32 value of its earlier position (see tests/coastcases.py)
    tol = 5e-7 if 'previous' in case else TOL_DEG
    err = 0.0
    for a, b in (('lon', 'lat'), ('d_lon', 'd_lat'), ('h_lon', 'h_lat')):
        if len(got[a]):
            err = max(err, *common.max_err_deg(got[a], got[b], g(a), g(b)))
    assert err < tol, (case, err)
    ztol = 1e-5 if case in WIND_K else 1e-9
    if exact_z and case not in RANDOMWALK:
        ztol = 0.0
    zerr = 0.0
    for k in ('z', 'd_z', 'h_z'):
        if len(got[k]):
            zerr = max(zerr, _zdiff(got[k], g(k)))
    assert zerr <= ztol, (case, zerr)
    return err, zerr


if __name__ == '__main__':
    from oracle import refrun
    refrun.setup()
    from opendrift.models.plastdrift import PlastDrift as RefPlast
    out = {}
    for case in CASES:
        ro = run_case(case, RefPlast, lambda lon, lat, z, t, f, name: refrun.make_grid_reader(lon, lat, z, t, f, name=name),
                      ref_update=RefPlast.update if case == 'subclass_reference_update' else None, logfile='/tmp/od_plast.log')
        s = summary(ro)
        for k, v in s.items():
            out['%s__%s' % (case, k)] = v
        print(case, 'active', len(s['id']), 'deactivated', len(s['d_id']), 'categories', list(s['cats']),
              'z float64 after each step', s['h_zf64'].astype(int).tolist(), 'z range %.3g .. %.3g' % (s['h_z'].min(), s['h_z'].max()))
    lon, lat = run_shear(RefPlast)
    out['shear__lon'], out['shear__lat'] = lon, lat
    print('test_wind_drift_shear without the landmask:', lon, lat, 'expected lon', SHEAR_LON)
    np.savez_compressed(GOLDEN, **out)
    print('wrote', GOLDEN)
