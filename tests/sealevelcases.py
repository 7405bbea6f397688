"""A varying sea surface height in OceanDrift (a sea_surface_height reader or a non-zero constant): the water column
sea_floor_depth + sea_surface_height in the sea-floor interaction, buoyancy and vertical mixing, and
drift:vertical_advection_correction with the previous-step store of sea_surface_height -- cases shared by the CPU (host engine)
and GPU tests.  The expected results come from the UNMODIFIED reference: tests/golden/sealevel_ref.npz, written by
`python tests/sealevelcases.py` (oracle/refrun.py).  The sea floor and the sea surface height are formulas on the current's grid."""
import os
from datetime import timedelta

import numpy as np

import common

GOLDEN = os.path.join(common.GOLDEN, 'sealevel_ref.npz')
N, STEPS = 400, 6

_RK2, _RK4 = {'drift:advection_scheme': 'runge-kutta'}, {'drift:advection_scheme': 'runge-kutta4'}
_CORR = dict(_RK4, **{'drift:vertical_advection_correction': True})
# name -> (config, readers among 'floor' / 'ssh' / 'k', terminal velocity, release over steps, sign of the time step)
CASES = {
    'lift_rk2': (dict(_RK2, **{'general:seafloor_action': 'lift_to_seafloor'}), ('floor', 'ssh'), -0.01, 0, 1),
    'deactivate_rk2': (dict(_RK2, **{'general:seafloor_action': 'deactivate'}), ('floor', 'ssh'), -0.01, 0, 1),
    'previous_rk2': (dict(_RK2, **{'general:seafloor_action': 'previous'}), ('floor', 'ssh'), -0.01, 0, 1),
    'constant_ssh': (dict(_RK2, **{'environment:constant:sea_surface_height': 0.6}), ('floor',), -0.01, 0, 1),
    'mixing': (dict(_RK4, **{'drift:vertical_mixing': True}), ('floor', 'ssh', 'k'), -0.002, 0, 1),
    'mixing_bottom_hook': (dict(_RK4, **{'drift:vertical_mixing': True}), ('floor', 'ssh', 'k'), -0.002, 0, 1),
    'correction_rk4': (_CORR, ('floor', 'ssh'), 0.0, 0, 1),
    'correction_fallback_floor': (_CORR, ('ssh',), 0.0, 0, 1),
    'correction_release_east': (dict(_CORR, **{'drift:deactivate_east_of': 3.3}), ('floor', 'ssh'), 0.0, 4, 1),
    'correction_backward': (_CORR, ('floor', 'ssh'), 0.0, 0, -1),
    'default_ssh_only': ({}, ('ssh',), 0.0, 0, 1),
    # the land mask from a gridded reader instead of a constant: an element whose depth became undefined is not covered by it either
    'correction_release_east_mask': (dict(_CORR, **{'drift:deactivate_east_of': 3.3, 'general:coastline_action': 'none'}),
                                     ('floor', 'ssh', 'mask'), 0.0, 4, 1),
    'correction_release_stranding': (dict(_CORR, **{'general:coastline_action': 'stranding',
                                                    'general:coastline_approximation_precision': None}),
                                     ('floor', 'ssh', 'mask'), 0.0, 4, 1),
    # a subclass whose update() reads environment_previous.sea_surface_height, as one written for the reference does
    'environment_previous_subclass': (dict(_CORR, **{'drift:deactivate_east_of': 3.3}), ('floor', 'ssh'), 0.0, 4, 1),
}
# depths that pass through the mixing kernel or the corrected vertical advection are compared to 1e-9 m; the others only see
# float32 environment arithmetic and Runge-Kutta sampling depths, compared to check_od's 1e-5 m like the other end-to-end cases
TIGHT_Z = ('mixing', 'mixing_bottom_hook', 'correction_rk4', 'correction_fallback_floor', 'correction_release_east',
           'correction_backward', 'correction_release_east_mask', 'correction_release_stranding', 'environment_previous_subclass')


def fields(fx):
    """(floor [ny, nx], ssh [nt, ny, nx]) float32 on the fixture's grid: a floor shoaling towards the east (15 .. 45 m), a sea
    surface height of +-0.8 m travelling west."""
    X, Y = np.meshgrid(fx.grid_lon, fx.grid_lat)
    xs = (X - fx.grid_lon[0]) / (fx.grid_lon[-1] - fx.grid_lon[0])
    floor = (45.0 - 30.0 * xs + 3.0 * np.sin(9.0 * Y)).astype(np.float32)
    ssh = np.stack([0.8 * np.sin(0.7 * k + 3.0 * X) for k in range(len(fx.times))]).astype(np.float32)
    return floor, ssh


def run_case(case, Model, make_reader, extra_config=None, **model_kw):
    """The same script on the reference's classes (generator) and on the product's."""
    cfg, readers, tv, release, sign = CASES[case]
    cfg = dict(cfg, **(extra_config or {}))
    fx = common.Fixture('rk4_3d_full')
    floor, ssh = fields(fx)
    if case == 'mixing_bottom_hook':
        class Hooked(Model):
            def bottom_interaction(self, Zmin=None):
                self.zmins.append(np.array(Zmin, dtype=np.float64))
        Model = Hooked
    if case == 'environment_previous_subclass':
        class Recorder(Model):
            def update(self):
                ep = self.environment_previous
                self.prev_ssh.append(np.array(np.asarray(ep.sea_surface_height), dtype=np.float64))
                self.prev_id.append(np.array(self.elements.ID, dtype=np.int64))
                super().update()
        Model = Recorder
    o = Model(loglevel=50, **model_kw)
    o.zmins, o.prev_ssh, o.prev_id = [], [], []
    comps = {common.CUR[0]: fx.u, common.CUR[1]: fx.v, 'upward_sea_water_velocity': (20.0 * fx.w).astype(np.float32)}
    if 'k' in readers:
        comps['ocean_vertical_diffusivity'] = common.Fixture('rk4_3d_mixing').kdiff
    o.add_reader(make_reader(fx.grid_lon, fx.grid_lat, fx.grid_z, fx.times, comps, 'current'))
    nt = len(fx.times)
    if 'floor' in readers:
        o.add_reader(make_reader(fx.grid_lon, fx.grid_lat, None, fx.times,
                                 {'sea_floor_depth_below_sea_level': np.repeat(floor[None], nt, axis=0)}, 'floor'))
    if 'ssh' in readers:
        o.add_reader(make_reader(fx.grid_lon, fx.grid_lat, None, fx.times, {'sea_surface_height': ssh}, 'ssh'))
    config = {'general:use_auto_landmask': False, 'seed:ocean_only': False, 'environment:constant:land_binary_mask': 0}
    if 'mask' in readers:        # land in the easternmost columns of the grid
        mask = np.zeros((len(fx.grid_lat), len(fx.grid_lon)), dtype=np.float32)
        mask[:, fx.grid_lon > 3.5] = 1.0
        o.add_reader(make_reader(fx.grid_lon, fx.grid_lat, None, fx.times, {'land_binary_mask': np.repeat(mask[None], nt, axis=0)}, 'mask'))
        config['environment:constant:land_binary_mask'] = None
    config.update(cfg)
    for k, val in config.items():
        o.set_config(k, val)
    if sign > 0:
        t = fx.start if not release else [fx.start, fx.start + timedelta(seconds=release * abs(fx.dt))]
    else:
        t = fx.times[-1] if not release else [fx.times[-1] - timedelta(seconds=release * abs(fx.dt)), fx.times[-1]]
    z = np.maximum(fx.z0[:N], np.float32(-40.0))
    o.seed_elements(lon=fx.lon0[:N], lat=fx.lat0[:N], z=z, time=t, terminal_velocity=tv)
    o.run(steps=STEPS, time_step=sign * abs(fx.dt), time_step_output=sign * abs(fx.dt))
    return o


def run_product(case, extra_config=None, **model_kw):
    from opendrift_b200.models.oceandrift import OceanDrift
    from opendrift_b200.readers import reader_regular_grid
    return run_case(case, OceanDrift, lambda lon, lat, z, t, f, name: reader_regular_grid.Reader(lon, lat, z, t, f, name=name),
                    extra_config, **model_kw)


def summary(o):
    el, de = o.elements, o.elements_deactivated
    out = {'id': np.asarray(el.ID, dtype=np.int64), 'lon': np.asarray(el.lon, dtype=np.float64), 'lat': np.asarray(el.lat, dtype=np.float64),
           'z': np.asarray(el.z, dtype=np.float64), 'cats': np.array(list(o.status_categories))}
    if o.num_elements_deactivated():
        out.update({'d_id': np.asarray(de.ID, dtype=np.int64), 'd_lon': np.asarray(de.lon, dtype=np.float64),
                    'd_lat': np.asarray(de.lat, dtype=np.float64), 'd_z': np.asarray(de.z, dtype=np.float64),
                    'd_status': np.asarray(de.status, dtype=np.int64)})
    else:
        out.update({'d_id': np.zeros(0, np.int64), 'd_lon': np.zeros(0), 'd_lat': np.zeros(0), 'd_z': np.zeros(0),
                    'd_status': np.zeros(0, np.int64)})
    zm = getattr(o, 'zmins', [])
    out['zmin'] = np.concatenate(zm) if zm else np.zeros(0)
    pv = getattr(o, 'prev_ssh', [])
    out['prev_ssh'] = np.concatenate(pv) if pv else np.zeros(0)
    out['prev_id'] = np.concatenate(o.prev_id) if pv else np.zeros(0, np.int64)
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
    assert np.array_equal(got['id'], g('id'))
    assert np.array_equal(got['d_id'], g('d_id'))                # same elements, same (concatenation) order
    assert np.array_equal(got['d_status'], g('d_status'))
    # 'previous': an element moved back lands on the float32 value of its earlier position (see tests/coastcases.py)
    tol = 5e-7 if 'previous' in case else 5e-8
    ztol = 1e-9 if case in TIGHT_Z else 1e-5
    if len(got['id']):
        assert max(common.max_err_deg(got['lon'], got['lat'], g('lon'), g('lat'))) < tol
        assert _zdiff(got['z'], g('z')) <= ztol, _zdiff(got['z'], g('z'))
    if len(got['d_id']):
        assert max(common.max_err_deg(got['d_lon'], got['d_lat'], g('d_lon'), g('d_lat'))) < tol
        assert _zdiff(got['d_z'], g('d_z')) <= ztol
    assert got['zmin'].shape == g('zmin').shape and np.array_equal(got['zmin'], g('zmin'))
    assert np.array_equal(got['prev_id'], g('prev_id'))
    assert np.array_equal(got['prev_ssh'], g('prev_ssh'), equal_nan=True)
    return len(got['id']), len(got['d_id']), list(got['cats'])


if __name__ == '__main__':
    from oracle import refrun
    refrun.setup()
    from opendrift.models.oceandrift import OceanDrift as RefOD
    out = {}
    for case in CASES:
        ro = run_case(case, RefOD, lambda lon, lat, z, t, f, name: refrun.make_grid_reader(lon, lat, z, t, f, name=name),
                      logfile='/tmp/od_sealevel.log')
        s = summary(ro)
        for k, v in s.items():
            out['%s__%s' % (case, k)] = v
        codes = {c: int((s['d_status'] == i).sum()) for i, c in enumerate(s['cats'])}
        print(case, 'active', len(s['id']), 'deactivated', len(s['d_id']), codes, 'NaN z', int(np.isnan(s['z']).sum()),
              'zmin calls', len(s['zmin']))
    np.savez_compressed(GOLDEN, **out)
    print('wrote', GOLDEN)
