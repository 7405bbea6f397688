"""drift:use_tabularised_stokes_drift in OceanDrift: the Stokes drift and the significant wave height estimated from the wind
with the reference's fetch tables -- cases shared by the CPU (host engine) and GPU tests.  The expected results come from the
UNMODIFIED reference: tests/golden/stokes_tab_ref.npz, written by `python tests/stokestabcases.py` (oracle/refrun.py).
Besides the positions and depths at the end of each run, the values that the public Environment.get_environment returns there
for the wind, the Stokes drift and the wave height are stored."""
import os

import numpy as np

import common

GOLDEN = os.path.join(common.GOLDEN, 'stokes_tab_ref.npz')
N, STEPS, DT = 400, 6, 900
SX, SY, HS = 'sea_surface_wave_stokes_drift_x_velocity', 'sea_surface_wave_stokes_drift_y_velocity', 'sea_surface_wave_significant_height'
ENV_VARS = ['x_wind', 'y_wind', SX, SY, HS]

_TAB = {'drift:advection_scheme': 'runge-kutta4', 'drift:use_tabularised_stokes_drift': True}
# name -> (config, readers among 'wind' / 'strong_wind' / 'hs' / 'stokes_pos' / 'stokes_le0', sign of the time step)
CASES = {
    'fetch5000': (dict(_TAB, **{'drift:tabularised_stokes_drift_fetch': '5000'}), ('wind',), 1),
    'fetch25000': (dict(_TAB, **{'drift:tabularised_stokes_drift_fetch': '25000'}), ('wind',), 1),
    'fetch50000': (dict(_TAB, **{'drift:tabularised_stokes_drift_fetch': '50000'}), ('wind',), 1),
    'monochromatic': (dict(_TAB, **{'drift:stokes_drift_profile': 'monochromatic'}), ('wind',), 1),
    'exponential': (dict(_TAB, **{'drift:stokes_drift_profile': 'exponential'}), ('wind',), 1),
    'hs_reader': (_TAB, ('wind', 'hs'), 1),
    'stokes_reader_positive': (_TAB, ('wind', 'stokes_pos'), 1),
    # every sample <= 0 and some exactly 0: max == 0, so the reader's Stokes drift is replaced (the reference's test)
    'stokes_reader_nonpositive': (_TAB, ('wind', 'stokes_le0'), 1),
    'wind_above_30': (_TAB, ('strong_wind',), 1),
    # the wind noise is drawn after the parameterisation, which sees the wind without it
    'wind_uncertainty': (dict(_TAB, **{'drift:wind_uncertainty': 2.0}), ('wind',), 1),
    'helper_subclass': (_TAB, ('wind',), 1),
    'constant_wind': (dict(_TAB, **{'environment:constant:x_wind': 7.5, 'environment:constant:y_wind': -4.25}), (), 1),
    'backward': (_TAB, ('wind',), -1),
    'mixing_wind': (dict(_TAB, **{'drift:vertical_mixing': True, 'vertical_mixing:diffusivitymodel': 'windspeed_Large1994'}),
                    ('wind',), 1),
}
# the public get_environment of the reference also adds the wind noise to the wind it returns
NOISY_WIND = ('wind_uncertainty',)


def fields(fx):
    """(positive Stokes drift x, y; non-positive Stokes drift x, y with a zero western half; Hs) [nt, ny, nx] float32 on the
    fixture's grid."""
    nt = len(fx.times)
    X, Y = np.meshgrid(fx.grid_lon, fx.grid_lat)
    pos_x = np.stack([0.08 + 0.04 * np.sin(0.5 * k + 2.0 * X) for k in range(nt)]).astype(np.float32)
    pos_y = np.stack([0.05 + 0.03 * np.cos(0.4 * k + 5.0 * Y) for k in range(nt)]).astype(np.float32)
    west = X < 0.5 * (fx.grid_lon[0] + fx.grid_lon[-1])
    le0_x = np.stack([np.where(west, 0.0, -0.06 * (1.2 + np.sin(0.5 * k + 2.0 * X))) for k in range(nt)]).astype(np.float32)
    le0_y = np.stack([np.where(west, 0.0, -0.04 * (1.1 + np.cos(0.4 * k + 5.0 * Y))) for k in range(nt)]).astype(np.float32)
    hs = np.stack([1.5 + 0.8 * np.sin(0.3 * k + 3.0 * X + Y) for k in range(nt)]).astype(np.float32)
    return pos_x, pos_y, le0_x, le0_y, hs


def run_case(case, Model, make_reader, extra_config=None, **model_kw):
    """The same script on the reference's classes (generator) and on the product's."""
    cfg, readers, sign = CASES[case]
    cfg = dict(cfg, **(extra_config or {}))
    fx = common.Fixture('rk4_3d_full')
    pos_x, pos_y, le0_x, le0_y, hs = fields(fx)
    if case == 'helper_subclass':
        class Helper(Model):
            def update(self):
                super().update()
        Model = Helper
    np.random.seed(11)
    o = Model(loglevel=50, **model_kw)
    o.add_reader(make_reader(fx.grid_lon, fx.grid_lat, fx.grid_z, fx.times,
                             {common.CUR[0]: fx.u, common.CUR[1]: fx.v, 'upward_sea_water_velocity': (20.0 * fx.w).astype(np.float32)},
                             'current'))
    grid2d = lambda f, name: make_reader(fx.grid_lon, fx.grid_lat, None, fx.times, f, name)       # noqa: E731
    if 'wind' in readers:
        o.add_reader(make_reader(fx.wind_lon, fx.wind_lat, None, fx.times, {'x_wind': fx.x_wind, 'y_wind': fx.y_wind}, 'wind'))
    if 'strong_wind' in readers:     # up to 39 m/s
        o.add_reader(make_reader(fx.wind_lon, fx.wind_lat, None, fx.times,
                                 {'x_wind': (3.0 * fx.x_wind).astype(np.float32), 'y_wind': (3.0 * fx.y_wind).astype(np.float32)},
                                 'wind'))
    if 'hs' in readers:
        o.add_reader(grid2d({HS: hs}, 'waves'))
    if 'stokes_pos' in readers:
        o.add_reader(grid2d({SX: pos_x, SY: pos_y}, 'stokes'))
    if 'stokes_le0' in readers:
        o.add_reader(grid2d({SX: le0_x, SY: le0_y}, 'stokes'))
    config = {'general:use_auto_landmask': False, 'seed:ocean_only': False, 'environment:constant:land_binary_mask': 0}
    config.update(cfg)
    for k, val in config.items():
        o.set_config(k, val)
    t = fx.start if sign > 0 else fx.times[-1]
    z = np.maximum(fx.z0[:N], np.float32(-20.0))
    o.seed_elements(lon=fx.lon0[:N], lat=fx.lat0[:N], z=z, time=t)
    o.run(steps=STEPS, time_step=sign * DT, time_step_output=sign * DT)
    el = o.elements
    env, _, _ = o.env.get_environment(ENV_VARS, o.time, np.asarray(el.lon), np.asarray(el.lat), np.asarray(el.z))
    o.stokes_tab_env = {v: np.array(env[v], dtype=np.float32) for v in ENV_VARS}
    return o


def run_product(case, extra_config=None, **model_kw):
    from opendrift_b200.models.oceandrift import OceanDrift
    from opendrift_b200.readers import reader_regular_grid
    return run_case(case, OceanDrift, lambda lon, lat, z, t, f, name: reader_regular_grid.Reader(lon, lat, z, t, f, name=name),
                    extra_config, **model_kw)


def summary(o):
    el = o.elements
    out = {'id': np.asarray(el.ID, dtype=np.int64), 'lon': np.asarray(el.lon, dtype=np.float64),
           'lat': np.asarray(el.lat, dtype=np.float64), 'z': np.asarray(el.z, dtype=np.float64),
           'n_deactivated': np.int64(o.num_elements_deactivated())}
    for v in ENV_VARS:
        out['env_' + v] = o.stokes_tab_env[v]
    return out


def check(o, case):
    ref = np.load(GOLDEN)
    got = summary(o)
    g = lambda k: ref['%s__%s' % (case, k)]                      # noqa: E731
    assert np.array_equal(got['id'], g('id'))
    assert int(got['n_deactivated']) == int(g('n_deactivated'))
    assert max(common.max_err_deg(got['lon'], got['lat'], g('lon'), g('lat'))) < 5e-8
    # depths to the 1e-5 m of the other end-to-end cases: the Large et al. (1994) mixing from the wind differs from the
    # reference by about 1e-6 m with or without this option
    assert np.max(np.abs(got['z'] - g('z'))) <= 1e-5, np.max(np.abs(got['z'] - g('z')))
    for v in ENV_VARS:
        if case in NOISY_WIND and v in ('x_wind', 'y_wind'):
            continue
        assert np.array_equal(got['env_' + v], g('env_' + v), equal_nan=True), v
    return len(got['id'])


if __name__ == '__main__':
    from oracle import refrun
    refrun.setup()
    from opendrift.models.oceandrift import OceanDrift as RefOD
    out = {}
    for case in CASES:
        ro = run_case(case, RefOD, lambda lon, lat, z, t, f, name: refrun.make_grid_reader(lon, lat, z, t, f, name=name),
                      logfile='/tmp/od_stokestab.log')
        s = summary(ro)
        for k, v in s.items():
            out['%s__%s' % (case, k)] = v
        print(case, 'active', len(s['id']), 'max |us|', float(np.nanmax(np.abs(s['env_' + SX]))),
              'max Hs', float(np.nanmax(s['env_' + HS])))
    np.savez_compressed(GOLDEN, **out)
    print('wrote', GOLDEN)
