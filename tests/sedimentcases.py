"""SedimentDrift: settling inside the mixing loop and resuspension -- cases shared by the CPU (host engine) and GPU tests.  The
expected results come from the UNMODIFIED reference's SedimentDrift: tests/golden/sediment_ref.npz, written by
`python tests/sedimentcases.py` (oracle/refrun.py).  Every run records, after each update(), the IDs, depths and moving flags of
the active elements; the end state includes the deactivated elements in the order they were removed."""
import os
from datetime import timedelta

import numpy as np

import common

GOLDEN = os.path.join(common.GOLDEN, 'sediment_ref.npz')
N, STEPS = 300, 8

_BASE = {'general:use_auto_landmask': False, 'seed:ocean_only': False, 'environment:constant:land_binary_mask': 0,
         'general:coastline_action': 'none', 'drift:advection_scheme': 'runge-kutta4'}
_LIFT = {'general:seafloor_action': 'lift_to_seafloor', 'vertical_mixing:resuspension_threshold': 0.3}
# the resuspension example's configuration (example_sediments_resuspension.py), in-memory readers
_EXAMPLE = {'environment:fallback:y_wind': -6, 'environment:fallback:x_wind': -3, 'environment:fallback:sea_floor_depth_below_sea_level': 30,
            'vertical_mixing:resuspension_threshold': .5, 'drift:current_uncertainty': 0.1, 'drift:wind_uncertainty': 1,
            'vertical_mixing:diffusivitymodel': 'windspeed_Large1994'}
_K0 = {'vertical_mixing:diffusivitymodel': 'constant', 'environment:fallback:ocean_vertical_diffusivity': 0.0,
       'environment:fallback:sea_floor_depth_below_sea_level': 30, 'drift:vertical_advection': False}
# name -> (config, readers among 'osc' / 'cur' / 'tidal' / 'k' / 'floor' / 'ssh' / 'mask' / 'wind', terminal velocity, release,
#          time step in seconds (negative: backward))
CASES = {
    'example_fallback_floor': (_EXAMPLE, ('osc',), -0.01, True, 1800),
    'example_glomma': (dict(_EXAMPLE, **{'drift:current_uncertainty': .2, 'drift:wind_uncertainty': 2}), ('osc',), -0.001, True, 600),
    'lift_profile': (_LIFT, ('tidal', 'k', 'floor', 'ssh'), -0.005, False, 900),
    'deactivate_profile': (dict(_LIFT, **{'general:seafloor_action': 'deactivate'}), ('tidal', 'k', 'floor', 'ssh'), -0.005, False, 900),
    'tidal_sundby': (dict(_LIFT, **{'vertical_mixing:diffusivitymodel': 'windspeed_Sundby1983'}), ('tidal', 'floor', 'wind'), -0.01,
                     False, 900),
    # a current of exactly float32(0.2) everywhere: float32(speed) > float32(0.2) is False, so nothing is resuspended
    'speed_at_threshold_constant': (dict(_LIFT, **{'vertical_mixing:diffusivitymodel': 'constant', 'vertical_mixing:resuspension_threshold': 0.2,
                                                   'environment:fallback:x_sea_water_velocity': 0.2}), ('floor',), -0.01, False, 900),
    'euler_large1994': (dict(_LIFT, **{'drift:advection_scheme': 'euler', 'vertical_mixing:diffusivitymodel': 'windspeed_Large1994'}),
                        ('cur', 'floor', 'wind'), -0.01, True, 900),
    'backward': (_LIFT, ('tidal', 'k', 'floor', 'ssh'), -0.005, False, -900),
    'mask_previous': (dict(_LIFT, **{'general:coastline_action': 'previous', 'general:coastline_approximation_precision': None,
                                     'environment:constant:land_binary_mask': None}), ('cur', 'floor', 'mask'), -0.01, True, 900),
    'mask_stranding': (dict(_LIFT, **{'general:coastline_action': 'stranding', 'general:coastline_approximation_precision': None,
                                      'environment:constant:land_binary_mask': None}), ('cur', 'floor', 'mask'), -0.01, True, 900),
    'hook_subclass': (_LIFT, ('tidal', 'floor'), -0.01, False, 900),
    # element 0 lies exactly on the (fallback) floor with K = 0 and w = 0: it settles only in an iteration where another element is
    # below the floor -- element 1 sinks there in the first iteration ('_sinker'), or never gets there ('_alone')
    'undecided_sinker': (_K0, (), None, False, 900),
    'undecided_alone': (_K0, (), None, False, 900),
}
# every case's depths pass through the mixing kernel: compared to 1e-9 m (sealevelcases.TIGHT_Z), except where the diffusivity
# comes from a wind that is not zero: the wind speed of the analytical models differs from the reference's by an ulp here and there
# (oceandrift.py's _mix), which moves depths by about 1e-6 m -- those are compared to the 1e-5 m of the other end-to-end cases
WIND_K = ('example_fallback_floor', 'example_glomma', 'tidal_sundby', 'euler_large1994')


def fields(fx):
    """(floor [ny, nx], ssh [nt, ny, nx], tidal u, v [nt, nz, ny, nx], mask [ny, nx]) float32 on the fixture's grid: a floor shoaling
    towards the east (15 .. 45 m), a sea surface height of +-0.8 m, a current whose speed crosses 0.3 m/s between the reader's times,
    land in the easternmost columns."""
    X, Y = np.meshgrid(fx.grid_lon, fx.grid_lat)
    xs = (X - fx.grid_lon[0]) / (fx.grid_lon[-1] - fx.grid_lon[0])
    floor = (45.0 - 30.0 * xs + 3.0 * np.sin(9.0 * Y)).astype(np.float32)
    nt, nz = len(fx.times), len(fx.grid_z)
    ssh = np.stack([0.8 * np.sin(0.7 * k + 3.0 * X) for k in range(nt)]).astype(np.float32)
    amp = [0.12, 0.42, 0.2, 0.5]
    u = np.stack([np.repeat((amp[k] * (1.0 + 0.3 * np.sin(2.0 * X + Y)))[None], nz, axis=0) for k in range(nt)]).astype(np.float32)
    v = (0.25 * u).astype(np.float32)
    mask = np.zeros(X.shape, dtype=np.float32)
    mask[:, fx.grid_lon > 3.5] = 1.0
    return floor, ssh, u, v, mask


def run_case(case, Model, make_reader, oscillating, extra_config=None, **model_kw):
    """The same script on the reference's classes (generator) and on the product's."""
    cfg, readers, tv, release, dt = CASES[case]
    cfg = dict(cfg, **(extra_config or {}))
    fx = common.Fixture('rk4_3d_full')
    floor, ssh, tu, tv_, mask = fields(fx)

    class Recorder(Model):
        def update(self):
            super().update()
            el = self.elements
            self.rec.append((np.array(el.ID, dtype=np.int64), np.array(el.z, dtype=np.float64), np.array(el.moving, dtype=np.int64)))

    if case == 'hook_subclass':
        class Hooked(Recorder):
            def bottom_interaction(self, seafloor_depth):          # the reference's body, and a record of each call
                self.n_hook += 1
                settling = np.logical_and(self.elements.z <= seafloor_depth, self.elements.moving == 1)
                if np.sum(settling) > 0:
                    self.elements.moving[settling] = 0
        Model = Hooked
    else:
        Model = Recorder
    np.random.seed(5)
    o = Model(loglevel=50, **model_kw)
    o.rec, o.n_hook = [], 0
    nt = len(fx.times)
    grid2d = lambda f, name: make_reader(fx.grid_lon, fx.grid_lat, None, fx.times, f, name)       # noqa: E731
    if 'osc' in readers:
        o.add_reader([oscillating.Reader('x_sea_water_velocity', amplitude=0.6, zero_time=fx.start),
                      oscillating.Reader('y_sea_water_velocity', amplitude=.3, period=timedelta(hours=5), zero_time=fx.start)])
    comps = {}
    if 'cur' in readers:
        comps = {common.CUR[0]: fx.u, common.CUR[1]: fx.v, 'upward_sea_water_velocity': (20.0 * fx.w).astype(np.float32)}
    if 'tidal' in readers:
        comps = {common.CUR[0]: tu, common.CUR[1]: tv_}
    if 'k' in readers:
        comps['ocean_vertical_diffusivity'] = common.Fixture('rk4_3d_mixing').kdiff
    if comps:
        o.add_reader(make_reader(fx.grid_lon, fx.grid_lat, fx.grid_z, fx.times, comps, 'current'))
    if 'wind' in readers:
        o.add_reader(make_reader(fx.wind_lon, fx.wind_lat, None, fx.times, {'x_wind': fx.x_wind, 'y_wind': fx.y_wind}, 'wind'))
    if 'floor' in readers:
        o.add_reader(grid2d({'sea_floor_depth_below_sea_level': np.repeat(floor[None], nt, axis=0)}, 'floor'))
    if 'ssh' in readers:
        o.add_reader(grid2d({'sea_surface_height': ssh}, 'ssh'))
    if 'mask' in readers:
        o.add_reader(grid2d({'land_binary_mask': np.repeat(mask[None], nt, axis=0)}, 'mask'))
    config = dict(_BASE)
    config.update(cfg)
    for k, val in config.items():
        o.set_config(k, val)
    t0 = fx.start if dt > 0 else fx.times[-1]
    t = [t0, t0 + timedelta(seconds=3 * dt)] if release else t0
    lon, lat = fx.lon0[:N], fx.lat0[:N]
    z = np.maximum(fx.z0[:N], np.float32(-40.0))
    if case.startswith('undecided'):
        lon, lat = lon[:4], lat[:4]
        z = np.array([-30.0, -29.9 if case.endswith('sinker') else -20.0, -10.0, -25.0], dtype=np.float32)
        tv = np.array([0.0, -0.01 if case.endswith('sinker') else 0.0, 0.0, 0.0], dtype=np.float32)
    o.seed_elements(lon=lon, lat=lat, z=z, time=t, terminal_velocity=tv)
    o.run(steps=STEPS, time_step=dt, time_step_output=dt)
    return o


def run_product(case, extra_config=None, **model_kw):
    from opendrift_b200.models.sedimentdrift import SedimentDrift
    from opendrift_b200.readers import reader_regular_grid, reader_oscillating
    return run_case(case, SedimentDrift, lambda lon, lat, z, t, f, name: reader_regular_grid.Reader(lon, lat, z, t, f, name=name),
                    reader_oscillating, extra_config, **model_kw)


def summary(o):
    el, de = o.elements, o.elements_deactivated
    out = {'id': np.asarray(el.ID, dtype=np.int64), 'lon': np.asarray(el.lon, dtype=np.float64), 'lat': np.asarray(el.lat, dtype=np.float64),
           'z': np.asarray(el.z, dtype=np.float64), 'moving': np.asarray(el.moving, dtype=np.int64),
           'status': np.asarray(el.status, dtype=np.int64), 'cats': np.array(list(o.status_categories)),
           'n_hook': np.int64(o.n_hook)}
    if o.num_elements_deactivated():
        out.update({'d_id': np.asarray(de.ID, dtype=np.int64), 'd_lon': np.asarray(de.lon, dtype=np.float64),
                    'd_lat': np.asarray(de.lat, dtype=np.float64), 'd_z': np.asarray(de.z, dtype=np.float64),
                    'd_status': np.asarray(de.status, dtype=np.int64), 'd_moving': np.asarray(de.moving, dtype=np.int64)})
    else:
        out.update({'d_id': np.zeros(0, np.int64), 'd_lon': np.zeros(0), 'd_lat': np.zeros(0), 'd_z': np.zeros(0),
                    'd_status': np.zeros(0, np.int64), 'd_moving': np.zeros(0, np.int64)})
    out['h_len'] = np.array([len(r[0]) for r in o.rec], dtype=np.int64)
    out['h_id'] = np.concatenate([r[0] for r in o.rec]) if o.rec else np.zeros(0, np.int64)
    out['h_z'] = np.concatenate([r[1] for r in o.rec]) if o.rec else np.zeros(0)
    out['h_moving'] = np.concatenate([r[2] for r in o.rec]) if o.rec else np.zeros(0, np.int64)
    return out


def _zdiff(a, b):
    """max |a - b| where both are finite; NaN depths must sit at the same places"""
    assert np.array_equal(np.isnan(a), np.isnan(b))
    f = ~np.isnan(a)
    return float(np.max(np.abs(a[f] - b[f]))) if f.any() else 0.0


def check(o, case):
    ref = np.load(GOLDEN)
    got = summary(o)
    g = lambda k: ref['%s__%s' % (case, k)]                      # noqa: E731
    assert list(got['cats']) == list(g('cats')), (list(got['cats']), list(g('cats')))
    for k in ('id', 'moving', 'status', 'd_id', 'd_status', 'd_moving', 'h_len', 'h_id', 'h_moving'):
        assert np.array_equal(got[k], g(k)), k
    assert int(got['n_hook']) == int(g('n_hook'))
    # 'previous': an element moved back lands on the float32 value of its earlier position (see tests/coastcases.py)
    tol = 5e-7 if 'previous' in case else 5e-8
    ztol = 1e-5 if case in WIND_K else 1e-9
    if len(got['id']):
        assert max(common.max_err_deg(got['lon'], got['lat'], g('lon'), g('lat'))) < tol
        assert _zdiff(got['z'], g('z')) <= ztol, _zdiff(got['z'], g('z'))
    if len(got['d_id']):
        assert max(common.max_err_deg(got['d_lon'], got['d_lat'], g('d_lon'), g('d_lat'))) < tol
        assert _zdiff(got['d_z'], g('d_z')) <= ztol
    assert _zdiff(got['h_z'], g('h_z')) <= ztol, _zdiff(got['h_z'], g('h_z'))
    return got


if __name__ == '__main__':
    from oracle import refrun
    refrun.setup()
    from opendrift.models.sedimentdrift import SedimentDrift as RefSD
    from opendrift.readers import reader_oscillating as ref_osc
    out = {}
    for case in CASES:
        ro = run_case(case, RefSD, lambda lon, lat, z, t, f, name: refrun.make_grid_reader(lon, lat, z, t, f, name=name), ref_osc,
                      logfile='/tmp/od_sediment.log')
        s = summary(ro)
        for k, v in s.items():
            out['%s__%s' % (case, k)] = v
        print(case, 'active', len(s['id']), 'settled', int((s['moving'] == 0).sum()), 'deactivated', len(s['d_id']),
              'settled in history', int((s['h_moving'] == 0).sum()), 'hook calls', int(s['n_hook']))
    np.savez_compressed(GOLDEN, **out)
    print('wrote', GOLDEN)
