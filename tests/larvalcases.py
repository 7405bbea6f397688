"""LarvalFish: cases shared by the CPU (host engine) and GPU tests.  The expected results come from the UNMODIFIED reference's
LarvalFish: tests/golden/larval_ref.npz, written by `python tests/larvalcases.py` (oracle/refrun.py).  Every run records, after each
update(), the IDs, positions and depths of the active elements with hatched, stage_fraction, weight, length and terminal_velocity,
and the dtype of each; the end state includes the deactivated elements in the order they were removed, with their status.  A run
whose update() raises records the error's type and the elements it leaves behind."""
import os
import zipfile
from datetime import datetime, timedelta

import numpy as np

import common

GOLDEN = os.path.join(common.GOLDEN, 'larval_ref.npz')
N, STEPS = 100, 8
VARS = ('z', 'hatched', 'stage_fraction', 'weight', 'length', 'terminal_velocity')

# the current's reader also serves a diffusivity profile of at least 0.02 m2/s, which keeps the elements, seeded at 5 .. 20 m,
# below the surface ('k3d': the profile as it is, 0.00015 .. 0.018 m2/s)
_BASE = {'general:use_auto_landmask': False, 'seed:ocean_only': False, 'environment:constant:land_binary_mask': 0,
         'general:coastline_action': 'none', 'vertical_mixing:diffusivitymodel': 'environment'}
_MASK = {'environment:constant:land_binary_mask': None, 'general:coastline_action': 'stranding',
         'general:coastline_approximation_precision': None}
# name -> (config, readers among 'cur' / 'ts' / 'k3d' / 'wind' / 'stokes' / 'floor' / 'mask', seeding ('scalar': the
#          defaults and a scalar depth; 'arrays': float32 arrays for every biology variable, half of them larvae, eggs close to
#          hatching; 'highre': arrays of diameters and salinities on both sides of the Reynolds limit; 'odd': hatched = 2 for all),
#          release over time, time step in seconds (negative: backward), hours the reader times are shifted by)
CASES = {
    'default_scalar': ({}, ('cur',), 'scalar', False, 900, 0),
    'ts_arrays_hatching': ({}, ('cur', 'ts'), 'arrays', False, 900, 0),
    'noon_crossing': ({}, ('cur', 'ts'), 'arrays', False, 900, 11),
    'high_reynolds': ({}, ('cur', 'ts'), 'highre', False, 900, 0),
    'diffusivity_reader': ({}, ('cur', 'k3d', 'ts'), 'arrays', False, 900, 0),
    'large1994_wind': ({'vertical_mixing:diffusivitymodel': 'windspeed_Large1994'}, ('cur', 'wind', 'ts'), 'arrays', False, 900, 0),
    'stokes_reader': ({'drift:stokes_drift_profile': 'exponential'}, ('cur', 'stokes', 'ts'), 'arrays', False, 900, 0),
    'no_mixing': ({'drift:vertical_mixing': False}, ('cur', 'ts'), 'arrays', False, 900, 0),
    'swim_0': ({'IBM:fraction_of_timestep_swimming': 0.0}, ('cur', 'ts'), 'arrays', False, 900, 0),
    'swim_1': ({'IBM:fraction_of_timestep_swimming': 1.0}, ('cur', 'ts'), 'arrays', False, 900, 0),
    'floor_lift': ({'general:seafloor_action': 'lift_to_seafloor'}, ('cur', 'floor'), 'arrays', False, 900, 0),
    'floor_deactivate': ({'general:seafloor_action': 'deactivate'}, ('cur', 'floor'), 'arrays', False, 900, 0),
    'mask_stranding': (_MASK, ('cur', 'mask'), 'arrays', True, 900, 0),
    'release_backward': ({}, ('cur', 'ts'), 'arrays', True, -900, 0),
    'uncertainty': ({'drift:current_uncertainty': 0.1}, ('cur', 'ts'), 'arrays', True, 900, 0),
    'hot_temperature': ({}, ('cur', 'ts'), 'arrays', False, 900, 0),
    'no_eggs_no_larvae': ({}, ('cur',), 'odd', False, 900, 0),
    'subclass_reference_update': ({}, ('cur', 'stokes', 'ts'), 'arrays', False, 900, 0),
    'fish_growth_subclass': ({}, ('cur', 'ts'), 'arrays', False, 900, 0),
}
# the reference's examples/example_larvae.py (run_example), shortened from 40 to EXAMPLE_DAYS days: long enough for every egg to
# hatch (about nine days at 10 degC) and for the larvae to swim through a few days and nights
EXAMPLE = 'example_larvae'
EXAMPLE_DAYS = 10
RAISES = ('hot_temperature', 'no_eggs_no_larvae')


def fields(fx):
    """float32 fields [nt, ny, nx] on the current grid: T of 4 .. 12 degC, S of 31.5 .. 34.5, Stokes drift towards the north-east,
    a shallow sea floor of 3 .. 12 m and land in the easternmost columns."""
    X, Y = np.meshgrid(fx.grid_lon, fx.grid_lat)
    xs = (X - fx.grid_lon[0]) / (fx.grid_lon[-1] - fx.grid_lon[0])
    nt = len(fx.times)
    rep = lambda a: np.repeat(a.astype(np.float32)[None], nt, axis=0)         # noqa: E731
    temp = np.stack([8.0 + 4.0 * np.sin(3.0 * X + 0.2 * k) for k in range(nt)]).astype(np.float32)
    salt = np.stack([33.0 + 1.5 * np.cos(2.0 * Y + 0.1 * k) for k in range(nt)]).astype(np.float32)
    sx = np.stack([0.05 + 0.1 * xs + 0.01 * k for k in range(nt)]).astype(np.float32)
    sy = rep(0.12 - 0.05 * np.sin(4.0 * Y))
    floor = rep(7.5 + 4.5 * np.sin(5.0 * X) * np.cos(4.0 * Y))
    mask = np.zeros(X.shape, dtype=np.float32)
    mask[:, fx.grid_lon > 3.6] = 1.0
    return temp, salt, sx, sy, floor, rep(mask)


def seeding(kind, n):
    """The biology keywords of seed_elements"""
    k = np.arange(n)
    if kind == 'scalar':
        return {'z': -10.0}
    z = (-5.0 - 15.0 * ((k * 7) % 23) / 22.0).astype(np.float32)
    if kind == 'odd':
        return {'z': z, 'hatched': np.full(n, 2, dtype=np.uint8)}
    kw = {'z': z, 'hatched': (k % 2).astype(np.uint8),
          'stage_fraction': (0.9 + 0.099 * ((k * 5) % 19) / 18.0).astype(np.float32),
          'weight': (0.05 + 0.4 * ((k * 3) % 11) / 10.0).astype(np.float32),
          'length': (4.0 + 2.0 * ((k * 7) % 5) / 4.0).astype(np.float32),
          'diameter': (0.0012 + 0.0004 * ((k * 11) % 7) / 6.0).astype(np.float32),
          'neutral_buoyancy_salinity': (31.0 + 1.0 * ((k * 13) % 9) / 8.0).astype(np.float32)}
    if kind == 'highre':
        # diameters of 0.3 .. 2 mm and neutral salinities of 30 .. 36: low and high Reynolds numbers, rising and sinking eggs
        kw['diameter'] = (0.0003 + 0.0017 * ((k * 11) % 13) / 12.0).astype(np.float32)
        kw['neutral_buoyancy_salinity'] = (30.0 + 6.0 * ((k * 13) % 17) / 16.0).astype(np.float32)
    return kw


def _record(o, rec):
    el = o.elements
    row = [np.array(el.ID, dtype=np.int64), np.array(el.lon, dtype=np.float64), np.array(el.lat, dtype=np.float64)]
    for v in VARS:
        a = np.atleast_1d(getattr(el, v))
        row.append((np.array(a, dtype=np.float64), str(a.dtype)))
    rec.append(row)


def run_case(case, Model, make_reader, extra_config=None, ref_update=None, growth=None, n=N, **model_kw):
    """The same script on the reference's classes and on the product's.  ref_update: the reference's LarvalFish.update, run by a
    subclass of Model (case 'subclass_reference_update'); growth: the reference's fish_growth, the override of a subclass (case
    'fish_growth_subclass').  Returns (model, the exception update() raised or None)."""
    cfg, readers, seed_kind, release, dt, shift = CASES[case]
    cfg = dict(cfg, **(extra_config or {}))
    fx = common.Fixture('rk4_3d_full')
    temp, salt, sx, sy, floor, mask = fields(fx)
    times = [t + timedelta(hours=shift) for t in fx.times]

    class Recorder(Model):
        def update(self):
            if case == 'hot_temperature':
                # the environment validates what readers give (T > 100 is missing data): a subclass heats every 7th element
                self.environment.sea_water_temperature[::7] = 101.0
            if ref_update is not None:
                ref_update(self)
            else:
                super().update()
            _record(self, self.rec)

    if growth is not None:
        Recorder.fish_growth = lambda self, weight, temperature: growth(self, weight, temperature)
    np.random.seed(17)
    o = Recorder(loglevel=50, **model_kw)
    o.rec = []
    grid2d = lambda f, name: make_reader(fx.grid_lon, fx.grid_lat, None, times, f, name)       # noqa: E731
    comps = {common.CUR[0]: fx.u, common.CUR[1]: fx.v}
    kdiff = common.Fixture('rk4_3d_mixing').kdiff
    comps['ocean_vertical_diffusivity'] = kdiff if 'k3d' in readers else np.maximum(kdiff, np.float32(0.02))
    o.add_reader(make_reader(fx.grid_lon, fx.grid_lat, fx.grid_z, times, comps, 'current'))
    if 'wind' in readers:
        o.add_reader(make_reader(fx.wind_lon, fx.wind_lat, None, times, {'x_wind': fx.x_wind, 'y_wind': fx.y_wind}, 'wind'))
    comps = {}
    if 'ts' in readers:
        comps.update({'sea_water_temperature': temp, 'sea_water_salinity': salt})
    if 'stokes' in readers:
        comps.update({'sea_surface_wave_stokes_drift_x_velocity': sx, 'sea_surface_wave_stokes_drift_y_velocity': sy})
    if 'floor' in readers:
        comps['sea_floor_depth_below_sea_level'] = floor
    if comps:
        o.add_reader(grid2d(comps, 'ocean'))
    if 'mask' in readers:
        o.add_reader(grid2d({'land_binary_mask': mask}, 'mask'))
    config = dict(_BASE)
    config.update(cfg)
    for k, val in config.items():
        o.set_config(k, val)
    t0 = times[0] if dt > 0 else times[-1]
    t = [t0, t0 + timedelta(seconds=3 * dt)] if release else t0
    o.seed_elements(lon=np.resize(fx.lon0, n), lat=np.resize(fx.lat0, n), time=t, number=n, **seeding(seed_kind, n))
    err = None
    try:
        o.run(steps=STEPS, time_step=dt, time_step_output=dt)
    except ValueError as e:
        err = e
    return o, err


def run_example(Model, Reader, days=EXAMPLE_DAYS):
    """examples/example_larvae.py of the reference with a run of `days` days: 20 eggs at rest in a constant reader (10 degC, a
    diffusivity of 0.02 m2/s), seeded with the defaults and released over 24 hours.  Returns (model, None)."""
    class Recorder(Model):
        def update(self):
            super().update()
            _record(self, self.rec)

    np.random.seed(3)
    o = Recorder(loglevel=50)
    o.rec = []
    o.add_reader(Reader({'x_sea_water_velocity': 0, 'y_sea_water_velocity': 0, 'x_wind': 0, 'y_wind': 0, 'sea_water_temperature': 10,
                         'land_binary_mask': 0, 'ocean_vertical_diffusivity': .02}))
    o.set_config('general:use_auto_landmask', False)
    time = datetime(2020, 7, 1, 12)
    o.seed_elements(lon=4, lat=60, time=[time, time + timedelta(hours=24)], number=20)
    o.run(duration=timedelta(days=days))
    return o, None


def run_product(case, extra_config=None, n=N, model=None, **model_kw):
    """model: a subclass of the product's LarvalFish to run in its place"""
    from opendrift_b200.models.larvalfish import LarvalFish
    from opendrift_b200.readers import reader_regular_grid, reader_constant
    if case == EXAMPLE:
        return run_example(model or LarvalFish, reader_constant.Reader)
    ref_update = growth = None
    if case in ('subclass_reference_update', 'fish_growth_subclass'):
        from oracle import refrun
        refrun.setup()
        from opendrift.models.larvalfish import LarvalFish as RefLarval
        ref_update = RefLarval.update if case == 'subclass_reference_update' else None
        growth = RefLarval.fish_growth if case == 'fish_growth_subclass' else None
    return run_case(case, model or LarvalFish, lambda lon, lat, z, t, f, name: reader_regular_grid.Reader(lon, lat, z, t, f, name=name),
                    extra_config, ref_update=ref_update, growth=growth, n=n, **model_kw)


def summary(o, err=None):
    el, de = o.elements, o.elements_deactivated
    out = {'id': np.asarray(el.ID, dtype=np.int64), 'lon': np.asarray(el.lon, dtype=np.float64), 'lat': np.asarray(el.lat, dtype=np.float64),
           'status': np.asarray(el.status, dtype=np.int64), 'cats': np.array(list(o.status_categories)),
           'error': np.array('' if err is None else type(err).__name__)}
    for v in VARS:
        a = np.atleast_1d(getattr(el, v))
        out[v] = np.array(a, dtype=np.float64)
        out[v + '_dtype'] = np.array(str(a.dtype))
    if o.num_elements_deactivated():
        out.update({'d_id': np.asarray(de.ID, dtype=np.int64), 'd_lon': np.asarray(de.lon, dtype=np.float64),
                    'd_lat': np.asarray(de.lat, dtype=np.float64), 'd_status': np.asarray(de.status, dtype=np.int64)})
    else:
        out.update({'d_id': np.zeros(0, np.int64), 'd_lon': np.zeros(0), 'd_lat': np.zeros(0), 'd_status': np.zeros(0, np.int64)})
    rec = o.rec
    out['h_len'] = np.array([len(r[0]) for r in rec], dtype=np.int64)
    cat = lambda j: np.concatenate([r[j] for r in rec]) if rec else np.zeros(0)            # noqa: E731
    out['h_id'], out['h_lon'], out['h_lat'] = cat(0).astype(np.int64), cat(1), cat(2)
    for j, v in enumerate(VARS):
        out['h_' + v] = np.concatenate([r[3 + j][0] for r in rec]) if rec else np.zeros(0)
        out['h_' + v + '_dtype'] = np.array([r[3 + j][1] for r in rec])
    return out


TOL_DEG = 5e-8
# Tolerances, relative to the value, by the dtype a quantity is computed in.  NumPy's float32 exp, log, log10 and pow are SIMD
# routines up to 2-3 ulp from the correctly rounded value; the launch uses the float64 functions rounded to float32 (half an ulp).
# A float32 result therefore differs by a few ulp of float32 (2^-23 = 1.2e-7) per call, and the weight grows by a sum of such
# terms each step: 2e-6 covers several steps of compounded 3-ulp differences.  In float64, glibc's functions and CUDA's differ by
# at most an ulp or two of float64 (2^-52 = 2.2e-16) per call.  Every chain starts from the float32 temperature, and a chain with a
# float32 exp / pow in it takes the float32 bound: the stage fraction (exp(3.65 - 0.145 T)) and the terminal velocity (exp and pow
# of float32 values in the high-Reynolds branch), whatever their own dtype.  A float64 weight meets only float32 products of T
# with constants, which both sides round alike; its log, pow and exp are float64.  Its growth and its length (computed in the
# weight's dtype) are therefore held to FLOW64_TOL where weight (and, for the length, length) are float64 throughout the run,
# compounded over the run's steps.  The depths: the mixing launch adds the buoyancy W * dt, up to about 1 m per step of 900 s, with
# W's relative difference (2e-6), and the larvae's swimming adds f * swim(L) * dt with that of swim(L): Z_TOL_STEP per step.
REL_TOL = {'float32': 2e-6, 'float64': 2e-6, 'uint8': 0.0}
FLOW64_TOL = 1e-12
Z_TOL_STEP = 2.5e-6


def _rel(a, b):
    """max |a - b| / max(|b|, tiny) where both are finite; NaN and infinite values must sit at the same places with the same values"""
    assert np.array_equal(np.isfinite(a), np.isfinite(b))
    assert np.array_equal(a[~np.isfinite(a)], b[~np.isfinite(b)], equal_nan=True)
    f = np.isfinite(a)
    if not f.any():
        return 0.0
    return float(np.max(np.abs(a[f] - b[f]) / np.maximum(np.abs(b[f]), 1e-30)))


def _abs(a, b):
    assert np.array_equal(np.isfinite(a), np.isfinite(b))
    f = np.isfinite(a)
    return float(np.max(np.abs(a[f] - b[f]))) if f.any() else 0.0


def compare(got, g, case):
    """got: summary() of a product run; g(k): the reference's.  Returns the largest differences found."""
    assert list(got['cats']) == list(g('cats')), (list(got['cats']), list(g('cats')))
    assert str(got['error']) == str(g('error')), (str(got['error']), str(g('error')))
    for k in ('id', 'status', 'd_id', 'd_status', 'h_len', 'h_id', 'hatched', 'h_hatched'):
        assert np.array_equal(got[k], g(k)), k
    for v in VARS:
        assert str(got[v + '_dtype']) == str(g(v + '_dtype')), (v, got[v + '_dtype'], g(v + '_dtype'))
        assert list(got['h_' + v + '_dtype']) == list(g('h_' + v + '_dtype')), v
    err = 0.0
    for a, b in (('lon', 'lat'), ('d_lon', 'd_lat'), ('h_lon', 'h_lat')):
        if len(got[a]):
            err = max(err, *common.max_err_deg(got[a], got[b], g(a), g(b)))
    assert err < TOL_DEG, (case, err)
    worst = {'pos': err}
    f64 = lambda v: len(g('h_len')) > 0 and all(str(d) == 'float64' for d in g('h_' + v + '_dtype'))        # noqa: E731
    for v in VARS[1:]:
        tol = max(REL_TOL[str(d)] for d in g('h_' + v + '_dtype')) if len(g('h_' + v + '_dtype')) else REL_TOL[str(g(v + '_dtype'))]
        if (v == 'weight' and f64('weight')) or (v == 'length' and f64('weight') and f64('length')):
            tol = FLOW64_TOL
        e = max(_rel(got[v], g(v)), _rel(got['h_' + v], g('h_' + v)))
        assert e <= tol, (case, v, e)
        worst[v] = e
    e = max(_abs(got['z'], g('z')), _abs(got['h_z'], g('h_z')))
    assert e <= Z_TOL_STEP * max(len(g('h_len')), 1), (case, 'z', e)
    worst['z'] = e
    return worst


def check(o, case, err=None):
    ref = np.load(GOLDEN)
    return compare(summary(o, err), lambda k: ref['%s__%s' % (case, k)], case)


def write_npz(path, arrays):
    """np.savez_compressed with a fixed date on every member, so that the same arrays give the same bytes"""
    with zipfile.ZipFile(path, 'w', compression=zipfile.ZIP_DEFLATED) as zf:
        for k, v in arrays.items():
            info = zipfile.ZipInfo(k + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            with zf.open(info, 'w') as f:
                np.lib.format.write_array(f, np.asanyarray(v), allow_pickle=False)


if __name__ == '__main__':
    from oracle import refrun
    refrun.setup()
    from opendrift.models.larvalfish import LarvalFish as RefLarval
    from opendrift.readers.reader_constant import Reader as RefConstant
    out = {}
    for case in CASES:
        ro, err = run_case(case, RefLarval, lambda lon, lat, z, t, f, name: refrun.make_grid_reader(lon, lat, z, t, f, name=name),
                           ref_update=RefLarval.update if case == 'subclass_reference_update' else None,
                           growth=RefLarval.fish_growth if case == 'fish_growth_subclass' else None, logfile='/tmp/od_larval.log')
        assert (err is not None) == (case in RAISES), (case, err)
        s = summary(ro, err)
        for k, v in s.items():
            out['%s__%s' % (case, k)] = v
        print(case, 'active', len(s['id']), 'deactivated', len(s['d_id']), 'categories', list(s['cats']), 'error', repr(err)[:60],
              'hatched', int((s['hatched'] == 1).sum()), 'dtypes', [str(s[v + '_dtype']) for v in VARS],
              'z %.3g .. %.3g' % (s['z'].min(), s['z'].max()) if len(s['z']) else '')
    ro, _ = run_example(RefLarval, RefConstant)
    for k, v in summary(ro).items():
        out['%s__%s' % (EXAMPLE, k)] = v
    print(EXAMPLE, 'hatched', int((np.asarray(ro.elements.hatched) == 1).sum()), 'of', len(ro.elements), 'z',
          np.asarray(ro.elements.z).min(), np.asarray(ro.elements.z).max())
    write_npz(GOLDEN, out)
    print('wrote', GOLDEN)
