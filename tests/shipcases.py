"""ShipDrift: cases shared by the CPU (host engine) and GPU tests.  The expected results come from the UNMODIFIED reference's ShipDrift:
tests/golden/ship_ref.npz, written by `python tests/shipcases.py` (oracle/refrun.py, the real scipy).  Every run records, after each
update(), the IDs and positions of the active elements; the end state includes the deactivated elements in the order they were
removed, with their status."""
import os
from datetime import timedelta

import numpy as np

import common

GOLDEN = os.path.join(common.GOLDEN, 'ship_ref.npz')
N, STEPS = 240, 8

_BASE = {'general:use_auto_landmask': False, 'seed:ocean_only': False, 'environment:constant:land_binary_mask': 0,
         'general:coastline_action': 'none'}
_D0 = {'environment:fallback:horizontal_diffusivity': 0}
_MASK = {'environment:constant:land_binary_mask': None}
# name -> (config, readers among 'cur' / 'wind' / 'wind_part' / 'wind_zero' / 'hs' / 'tm' / 'tm_part' / 'tp' / 'stokes' / 'mask',
#          ship sizes ('default' / 'mixed'), release over time, time step in seconds (negative: backward))
CASES = {
    'wind_only': (_D0, ('cur', 'wind'), 'default', False, 900),
    'waves_hs_tm02': (_D0, ('cur', 'wind', 'hs', 'tm'), 'mixed', False, 900),
    'tp_only': (_D0, ('cur', 'wind', 'tp'), 'default', False, 900),
    'tm02_partial': (_D0, ('cur', 'wind', 'hs', 'tm_part'), 'mixed', False, 900),
    'stokes_direction': (_D0, ('cur', 'wind', 'stokes'), 'mixed', False, 900),
    'zero_wind': (_D0, ('cur', 'wind_zero'), 'mixed', False, 900),
    'mask_none': (dict(_D0, **_MASK), ('cur', 'wind', 'mask'), 'default', False, 900),
    'mask_stranding': (dict(_D0, **_MASK, **{'general:coastline_action': 'stranding', 'general:coastline_approximation_precision': None}),
                       ('cur', 'wind', 'mask'), 'default', False, 900),
    'missing_wind': (_D0, ('cur', 'wind_part'), 'default', False, 900),
    'release_backward': (_D0, ('cur', 'wind', 'hs', 'tm'), 'mixed', True, -900),
    'diffusivity_default': ({}, ('cur', 'wind', 'hs', 'tm'), 'mixed', True, 900),
    'subclass_reference_update': (_D0, ('cur', 'wind', 'hs', 'tm_part', 'stokes'), 'mixed', False, 900),
}
TM02 = 'sea_surface_wave_mean_period_from_variance_spectral_density_second_frequency_moment'
TP = 'sea_surface_wave_period_at_variance_spectral_density_maximum'


def fields(fx):
    """float32 fields [nt, ny, nx] on the current grid: Hs of 0.5 .. 4.5 m, a period from 3 to 11 s across the grid (it crosses 5.7 and
    8.55 s, and takes those values exactly in two columns), Stokes drift towards the north-east, land in the easternmost columns."""
    X, Y = np.meshgrid(fx.grid_lon, fx.grid_lat)
    xs = (X - fx.grid_lon[0]) / (fx.grid_lon[-1] - fx.grid_lon[0])
    nt = len(fx.times)
    hs = np.stack([2.5 + 2.0 * np.sin(3.0 * X + 0.5 * k) * np.cos(5.0 * Y) for k in range(nt)]).astype(np.float32)
    tm = np.stack([3.0 + 8.0 * xs + 0.2 * k for k in range(nt)]).astype(np.float32)
    tm[:, :, 10] = np.float32(5.7)
    tm[:, :, 25] = np.float32(8.55)
    tm_part = tm.copy()
    tm_part[:, :, :14] = 0.0                                   # a wave model that covers part of the domain (fallback 0 elsewhere)
    sx = np.stack([0.05 + 0.1 * xs + 0.01 * k for k in range(nt)]).astype(np.float32)
    sy = np.stack([0.12 - 0.05 * np.sin(4.0 * Y) + 0.0 * k for k in range(nt)]).astype(np.float32)
    mask = np.zeros(X.shape, dtype=np.float32)
    mask[:, fx.grid_lon > 3.6] = 1.0
    return hs, tm, tm_part, sx, sy, np.repeat(mask[None], nt, axis=0)


def sizes(kind, n):
    """(length, height, draft, beam) float32: the defaults, or a mix of ship sizes in and out of the table's ranges (beam / length
    0.1 .. 0.2, draft / length 0.02 .. 0.08, exposed height below and above 15 and 37.2 m)."""
    if kind == 'default':
        return {}
    k = np.arange(n)
    length = (30.0 + (k * 37) % 270).astype(np.float32)
    beam = (length * (0.1 + 0.1 * ((k * 7) % 11) / 10.0)).astype(np.float32)
    draft = (length * (0.02 + 0.06 * ((k * 5) % 13) / 12.0)).astype(np.float32)
    height = (draft + 5.0 + (k * 3) % 45).astype(np.float32)
    return {'length': length, 'height': height, 'draft': draft, 'beam': beam}


def run_case(case, Model, make_reader, extra_config=None, ref_update=None, n=N, **model_kw):
    """The same script on the reference's classes and on the product's.  ref_update: the reference's ShipDrift.update, run by a
    subclass of Model (case 'subclass_reference_update').  n: ships (the fixture's start positions repeated)."""
    cfg, readers, kind, release, dt = CASES[case]
    cfg = dict(cfg, **(extra_config or {}))
    fx = common.Fixture('rk4_3d_full')
    hs, tm, tm_part, sx, sy, mask = fields(fx)

    class Recorder(Model):
        def update(self):
            if ref_update is not None:
                ref_update(self)
            else:
                super().update()
            el = self.elements
            self.rec.append((np.array(el.ID, dtype=np.int64), np.array(el.lon, dtype=np.float64), np.array(el.lat, dtype=np.float64)))

    np.random.seed(7)
    o = Recorder(loglevel=50, **model_kw)
    o.rec = []
    grid2d = lambda f, name: make_reader(fx.grid_lon, fx.grid_lat, None, fx.times, f, name)       # noqa: E731
    if 'cur' in readers:
        o.add_reader(make_reader(fx.grid_lon, fx.grid_lat, fx.grid_z, fx.times, {common.CUR[0]: fx.u, common.CUR[1]: fx.v}, 'current'))
    if 'wind' in readers or 'wind_zero' in readers:
        xw, yw = fx.x_wind.copy(), fx.y_wind.copy()
        if 'wind_zero' in readers:
            xw[:, :, ::3] = 0.0
            yw[:, :, ::3] = 0.0
        o.add_reader(make_reader(fx.wind_lon, fx.wind_lat, None, fx.times, {'x_wind': xw, 'y_wind': yw}, 'wind'))
    if 'wind_part' in readers:
        # the wind covers only the western part of the domain: elements that drift out of it leave as 'missing_data'
        o.add_reader(make_reader(fx.wind_lon[:22], fx.wind_lat, None, fx.times,
                                 {'x_wind': np.ascontiguousarray(fx.x_wind[:, :, :22]) + 6.0,
                                  'y_wind': np.ascontiguousarray(fx.y_wind[:, :, :22])}, 'wind'))
    comps = {}
    if 'hs' in readers:
        comps['sea_surface_wave_significant_height'] = hs
    if 'tm' in readers:
        comps[TM02] = tm
    if 'tm_part' in readers:
        comps[TM02] = tm_part
    if 'tp' in readers:
        comps[TP] = tm
    if 'stokes' in readers:
        comps['sea_surface_wave_stokes_drift_x_velocity'] = sx
        comps['sea_surface_wave_stokes_drift_y_velocity'] = sy
    if comps:
        o.add_reader(grid2d(comps, 'waves'))
    if 'mask' in readers:
        o.add_reader(grid2d({'land_binary_mask': mask}, 'mask'))
    config = dict(_BASE)
    config.update(cfg)
    for k, val in config.items():
        o.set_config(k, val)
    t0 = fx.start if dt > 0 else fx.start + timedelta(hours=2, minutes=30)
    t = [t0, t0 + timedelta(seconds=3 * dt)] if release else t0
    o.seed_elements(lon=np.resize(fx.lon0, n), lat=np.resize(fx.lat0, n), time=t, number=n, **sizes(kind, n))
    o.run(steps=STEPS, time_step=dt, time_step_output=dt)
    return o


def run_product(case, extra_config=None, n=N, **model_kw):
    from opendrift_b200.models.shipdrift import ShipDrift
    from opendrift_b200.readers import reader_regular_grid
    ref_update = None
    if case == 'subclass_reference_update':
        from oracle import refrun
        refrun.setup()
        from opendrift.models.shipdrift import ShipDrift as RefShip
        ref_update = RefShip.update
    model_kw.setdefault('wforce', wforce_path())
    return run_case(case, ShipDrift, lambda lon, lat, z, t, f, name: reader_regular_grid.Reader(lon, lat, z, t, f, name=name),
                    extra_config, ref_update=ref_update, n=n, **model_kw)


def wforce_path():
    """The reference's wforce.dat: the copy oracle/build_ref.py makes (travels with the tree), else the reference tree itself."""
    from oracle import refrun
    return os.path.join(refrun.REFERENCE_ROOT, 'opendrift', 'models', 'wforce.dat')


def summary(o):
    el, de = o.elements, o.elements_deactivated
    out = {'id': np.asarray(el.ID, dtype=np.int64), 'lon': np.asarray(el.lon, dtype=np.float64), 'lat': np.asarray(el.lat, dtype=np.float64),
           'status': np.asarray(el.status, dtype=np.int64), 'cats': np.array(list(o.status_categories))}
    if o.num_elements_deactivated():
        out.update({'d_id': np.asarray(de.ID, dtype=np.int64), 'd_lon': np.asarray(de.lon, dtype=np.float64),
                    'd_lat': np.asarray(de.lat, dtype=np.float64), 'd_status': np.asarray(de.status, dtype=np.int64)})
    else:
        out.update({'d_id': np.zeros(0, np.int64), 'd_lon': np.zeros(0), 'd_lat': np.zeros(0), 'd_status': np.zeros(0, np.int64)})
    out['h_len'] = np.array([len(r[0]) for r in o.rec], dtype=np.int64)
    out['h_id'] = np.concatenate([r[0] for r in o.rec]) if o.rec else np.zeros(0, np.int64)
    out['h_lon'] = np.concatenate([r[1] for r in o.rec]) if o.rec else np.zeros(0)
    out['h_lat'] = np.concatenate([r[2] for r in o.rec]) if o.rec else np.zeros(0)
    return out


TOL_DEG = 5e-8


def check(o, case):
    """Returns the largest position difference (degrees) against the reference."""
    ref = np.load(GOLDEN)
    got = summary(o)
    g = lambda k: ref['%s__%s' % (case, k)]                      # noqa: E731
    assert list(got['cats']) == list(g('cats')), (list(got['cats']), list(g('cats')))
    for k in ('id', 'status', 'd_id', 'd_status', 'h_len', 'h_id'):
        assert np.array_equal(got[k], g(k)), k
    err = 0.0
    for a, b in (('lon', 'lat'), ('d_lon', 'd_lat'), ('h_lon', 'h_lat')):
        if len(got[a]):
            err = max(err, *common.max_err_deg(got[a], got[b], g(a), g(b)))
    assert err < TOL_DEG, (case, err)
    return err


if __name__ == '__main__':
    from oracle import refrun
    refrun.setup()
    from opendrift.models.shipdrift import ShipDrift as RefShip
    out = {}
    for case in CASES:
        ro = run_case(case, RefShip, lambda lon, lat, z, t, f, name: refrun.make_grid_reader(lon, lat, z, t, f, name=name),
                      logfile='/tmp/od_ship.log')
        s = summary(ro)
        for k, v in s.items():
            out['%s__%s' % (case, k)] = v
        print(case, 'active', len(s['id']), 'deactivated', len(s['d_id']), 'categories', list(s['cats']))
    np.savez_compressed(GOLDEN, **out)
    print('wrote', GOLDEN)
