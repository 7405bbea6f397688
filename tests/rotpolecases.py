"""Gridded readers on a rotated-pole grid ('+proj=ob_tran +o_proj=longlat', the CF rotated_latitude_longitude mapping): the drop-in
model classes against runs of the UNMODIFIED reference on readers of the same grid -- cases shared by the CPU (host engine) and GPU
tests.  The expected results are tests/golden/rotpole_ref.npz, written by `python tests/rotpolecases.py` (oracle/refrun.py; the
reference's pyproj is its stand-in extended by oracle/proj_obtran.py, which tests/test_rotpole_host.py pins to the closed forms).

The grids are regular in rotated degrees.  Besides ordinary ones, two reproduce what the reference does with rotated longitudes it
takes for geographic ones: a grid west and east of rotated x = 0 whose TRUE corners all lie east of Greenwich (its elements west of
x = 0 are tested as x + 360 and get the fallback values), and grids whose rotated axis runs past 180 (x from 175 to 195: covered
and indexed mod 360 when the true corners are east of Greenwich, only the part up to 180 covered otherwise)."""
import os

import numpy as np

import common

GOLDEN = os.path.join(common.GOLDEN, 'rotpole_ref.npz')
N = 400
WAM = '+proj=ob_tran +o_proj=longlat +lon_0=-40 +o_lat_p=22 +R=6.371e+06 +no_defs'          # (the MyWave-WAM style grid)
ROT_EAST = '+proj=ob_tran +o_proj=longlat +o_lon_p=0 +o_lat_p=30 +lon_0=10 +R=6370997 +no_defs'
CROSS_EAST = '+proj=ob_tran +o_proj=longlat +o_lat_p=35 +o_lon_p=185 +lon_0=20 +R=6371000 +no_defs'
CROSS_GREENWICH = '+proj=ob_tran +o_proj=longlat +o_lat_p=35 +o_lon_p=185 +lon_0=0 +R=6371000 +no_defs'

_RK2, _RK4 = {'drift:advection_scheme': 'runge-kutta'}, {'drift:advection_scheme': 'runge-kutta4'}
_2D = {'drift:vertical_advection': False}
# name -> dict(proj4, model, readers, steps, dt, cfg, grid (x0, y0, dx, nx, ny), seed z)
CASES = {
    'wam_rk4_3d_w': dict(proj4=WAM, model='OceanDrift', readers=('cur3d',), steps=8, dt=600, cfg=_RK4),
    # current from a geographic reader, Stokes drift and wind from the rotated (wave / atmosphere) one
    'operational_rk2': dict(proj4=WAM, model='OceanDrift', readers=('geo_cur', 'stokes_wind'), steps=6, dt=900,
                            cfg=dict(_RK2, **_2D), z=0.0),
    'leeway': dict(proj4=WAM, model='Leeway', readers=('cur2d', 'wind'), steps=6, dt=600, cfg={}),
    'mixing_floor': dict(proj4=WAM, model='OceanDrift', readers=('cur3d_k', 'floor'), steps=3, dt=600,
                         cfg=dict(_2D, **{'drift:vertical_mixing': True, 'vertical_mixing:timestep': 60.0})),
    'fallback_west_of_0': dict(proj4=ROT_EAST, model='OceanDrift', readers=('cur2d',), steps=6, dt=900, cfg=dict(_RK2, **_2D),
                               grid=(-0.86, -0.74, 0.04, 44, 38), z=0.0, seed_margin=0),
    'cross_180_east': dict(proj4=CROSS_EAST, model='OceanDrift', readers=('cur2d', 'wind'), steps=6, dt=900, cfg=dict(_RK4, **_2D),
                           grid=(175.0, -5.0, 0.5, 41, 21), z=0.0, seed_margin=1),
    'cross_180_greenwich': dict(proj4=CROSS_GREENWICH, model='OceanDrift', readers=('cur2d',), steps=6, dt=900,
                                cfg=dict(_RK4, **_2D), grid=(175.0, -5.0, 0.5, 41, 21), z=0.0, seed_margin=1),
    'wam_backward_rk4': dict(proj4=WAM, model='OceanDrift', readers=('cur2d', 'wind'), steps=6, dt=-900, cfg=dict(_RK4, **_2D), z=0.0),
}


def setup(case):
    """The rotated grid, its fields, and the seeds (true lon / lat, float32) of one case."""
    from oracle.proj_obtran import ObTran
    c = CASES[case]
    P = ObTran(c['proj4'])
    if 'grid' in c:
        x0, y0, d, nx, ny = c['grid']
    else:
        cx, cy = P.forward_deg(np.array([4.0]), np.array([60.0]))
        nx, ny, d = 44, 38, 0.04
        x0, y0 = float(cx[0]) - d * (nx // 2), float(cy[0]) - d * (ny // 2)
    xs = (x0 + d * np.arange(nx)).astype(np.float32)
    ys = (y0 + d * np.arange(ny)).astype(np.float32)
    zs = -10.0 * np.arange(6)
    times = common.syn.slab_times(4)
    X, Y = np.meshgrid(np.linspace(0, 1, nx), np.linspace(0, 1, ny))
    lay = lambda fn: np.stack([[fn(k, z) for z in zs] for k in range(len(times))]).astype(np.float32)      # noqa: E731
    flat = lambda fn: np.stack([fn(k) for k in range(len(times))]).astype(np.float32)                      # noqa: E731
    U3 = lay(lambda k, z: 0.5 * np.sin(2 * np.pi * X + 0.3 * k) * np.cos(np.pi * Y) * np.exp(z / 40))
    V3 = lay(lambda k, z: 0.4 * np.cos(2 * np.pi * Y + 0.2 * k) * np.sin(np.pi * X) * np.exp(z / 40))
    wind = {'x_wind': flat(lambda k: 8 * np.cos(0.4 * k) * (1 + 0.3 * np.sin(np.pi * X))),
            'y_wind': flat(lambda k: 8 * np.sin(0.4 * k) * (1 + 0.3 * np.cos(np.pi * Y)))}
    fields = {
        'cur3d': {common.CUR[0]: U3, common.CUR[1]: V3,
                  'upward_sea_water_velocity': lay(lambda k, z: 1e-3 * np.sin(np.pi * X) * np.sin(np.pi * Y) * np.sin(np.pi * z / zs.min()))},
        'cur3d_k': {common.CUR[0]: U3, common.CUR[1]: V3,
                    'ocean_vertical_diffusivity': lay(lambda k, z: 0.01 * np.exp(z / 20) * (1 + 0.5 * np.sin(np.pi * X) * np.sin(np.pi * Y)))},
        'floor': {'sea_floor_depth_below_sea_level': flat(lambda k: 30.0 + 25.0 * X + 10.0 * Y)},
        'cur2d': {common.CUR[0]: U3[:, 0].copy(), common.CUR[1]: V3[:, 0].copy()},
        'wind': wind,
        'stokes_wind': dict(wind, **{'sea_surface_wave_stokes_drift_x_velocity': flat(lambda k: 0.15 * np.cos(0.3 * k + np.pi * Y)),
                                     'sea_surface_wave_stokes_drift_y_velocity': flat(lambda k: 0.1 * np.sin(0.3 * k + np.pi * X))}),
    }
    rng = np.random.default_rng(11)
    m = c.get('seed_margin', 3)
    px, py = rng.uniform(xs[m], xs[-1 - m], N), rng.uniform(ys[m], ys[-1 - m], N)
    lon0, lat0 = P.inverse_deg(px, py)
    z0 = np.full(N, c['z'], dtype=np.float32) if 'z' in c else rng.uniform(-35, 0, N).astype(np.float32)
    return c, xs, ys, zs, times, fields, lon0.astype(np.float32), lat0.astype(np.float32), z0


def geo_current(lon0, lat0, times):
    """A geographic current grid around the seeds (the ocean model of the operational combination)."""
    gl = np.arange(np.floor(lon0.min()) - 1, np.ceil(lon0.max()) + 1.01, 0.05).astype(np.float32)
    ga = np.arange(np.floor(lat0.min()) - 1, np.ceil(lat0.max()) + 1.01, 0.05).astype(np.float32)
    X, Y = np.meshgrid(np.linspace(0, 1, len(gl)), np.linspace(0, 1, len(ga)))
    u = np.stack([0.3 * np.sin(3 * np.pi * Y + 0.2 * k) for k in range(len(times))]).astype(np.float32)
    v = np.stack([0.25 * np.cos(3 * np.pi * X - 0.1 * k) for k in range(len(times))]).astype(np.float32)
    return gl, ga, {common.CUR[0]: u, common.CUR[1]: v}


def run_case(case, classes, make_reader, **model_kw):
    """make_reader(x, y, z, times, fields, name, proj4) -> a reader of the product or of the reference."""
    c, xs, ys, zs, times, fields, lon0, lat0, z0 = setup(case)
    o = classes[c['model']](loglevel=50, seed=0, **model_kw)
    for nm in c['readers']:
        if nm == 'geo_cur':
            gl, ga, f = geo_current(lon0, lat0, times)
            o.add_reader(make_reader(gl, ga, None, times, f, nm, '+proj=latlong'))
            continue
        o.add_reader(make_reader(xs, ys, zs if nm.startswith('cur3d') else None, times, fields[nm], nm, c['proj4']))
    for k, v in {'general:use_auto_landmask': False, 'general:coastline_action': 'none', **c['cfg']}.items():
        o.set_config(k, v)
    if 'environment:constant:land_binary_mask' in getattr(o, '_config', {}):
        o.set_config('environment:constant:land_binary_mask', 0)
    t0 = times[-1] if c['dt'] < 0 else times[0]
    if c['model'] == 'Leeway':
        o.seed_elements(lon=lon0, lat=lat0, time=t0, object_type=1)
    else:
        o.seed_elements(lon=lon0, lat=lat0, z=z0, time=t0)
    o.run(steps=c['steps'], time_step=c['dt'], time_step_output=abs(c['dt']))
    return o


def run_product(case, **model_kw):
    from opendrift_b200.models.oceandrift import OceanDrift
    from opendrift_b200.models.leeway import Leeway
    from opendrift_b200.readers import reader_regular_grid
    return run_case(case, {'OceanDrift': OceanDrift, 'Leeway': Leeway},
                    lambda x, y, z, t, f, name, proj4: reader_regular_grid.Reader(x, y, z, t, f, name=name, proj4=proj4), **model_kw)


def run_many(sort_every, n=120000):
    """n elements with the device generator on the WAM-style grid (3-D current with w, and wind): with sort_every = 1 the device
    arrays are sorted by the rotated grid's cells every step.  No reference run: the sorted run must equal the unsorted one."""
    from opendrift_b200.models.oceandrift import OceanDrift
    from opendrift_b200.readers import reader_regular_grid
    c, xs, ys, zs, times, fields, _, _, _ = setup('wam_rk4_3d_w')
    o = OceanDrift(loglevel=50)
    o.add_reader(reader_regular_grid.Reader(xs, ys, zs, times, fields['cur3d'], name='cur3d', proj4=WAM))
    o.add_reader(reader_regular_grid.Reader(xs, ys, None, times, fields['wind'], name='wind', proj4=WAM))
    for k, v in {'general:use_auto_landmask': False, 'environment:constant:land_binary_mask': 0, 'seed:ocean_only': False,
                 'general:coastline_action': 'none', 'drift:advection_scheme': 'runge-kutta4', 'gpu:rng': 'philox',
                 'gpu:sort_interval_steps': sort_every}.items():
        o.set_config(k, v)
    from oracle.proj_obtran import ObTran
    rng = np.random.default_rng(7)
    lon, lat = ObTran(WAM).inverse_deg(rng.uniform(xs[1], xs[-2], n), rng.uniform(ys[1], ys[-2], n))
    o.seed_elements(lon=lon, lat=lat, z=-rng.uniform(0, 40, n).astype(np.float32), time=times[0])
    o.run(steps=4, time_step=600, time_step_output=600)
    return o


def unmoved(lon, lat, lon0, lat0):
    """elements that never moved: those that got the fallback current on every step"""
    return int(np.sum((np.asarray(lon, dtype=np.float32) == lon0) & (np.asarray(lat, dtype=np.float32) == lat0)))


def check(o, case):
    """(max position error in degrees, max depth error in metres, how far the reference moved the elements)"""
    ref = np.load(GOLDEN)
    g = lambda k: ref['%s__%s' % (case, k)]                 # noqa: E731
    e = max(common.max_err_deg(np.asarray(o.elements.lon), np.asarray(o.elements.lat), g('lon'), g('lat')))
    dz = float(np.abs(np.asarray(o.elements.z, dtype=np.float64) - g('z')).max())
    moved = float(np.max(np.hypot(g('lon') - g('lon0'), g('lat') - g('lat0'))))
    return e, dz, moved


if __name__ == '__main__':
    from oracle import refrun, proj_obtran
    refrun.setup()
    proj_obtran.install()
    from opendrift.models.oceandrift import OceanDrift as RefOD
    from opendrift.models.leeway import Leeway as RefLW
    out = {}
    for case in CASES:
        ro = run_case(case, {'OceanDrift': RefOD, 'Leeway': RefLW},
                      lambda x, y, z, t, f, name, proj4: refrun.make_grid_reader(x, y, z, t, f, name=name, proj4=proj4),
                      logfile='/tmp/od_rotpole.log')
        lon0, lat0 = setup(case)[6:8]
        lon, lat = np.asarray(ro.elements.lon, dtype=np.float64), np.asarray(ro.elements.lat, dtype=np.float64)
        out.update({'%s__lon' % case: lon, '%s__lat' % case: lat, '%s__z' % case: np.asarray(ro.elements.z, dtype=np.float64),
                    '%s__lon0' % case: lon0.astype(np.float64), '%s__lat0' % case: lat0.astype(np.float64),
                    '%s__unmoved' % case: np.int64(unmoved(lon, lat, lon0, lat0))})
        print(case, len(lon), 'moved', float(np.max(np.hypot(lon - lon0, lat - lat0))), 'unmoved', unmoved(lon, lat, lon0, lat0))
    np.savez_compressed(GOLDEN, **out)
    print('wrote', GOLDEN)
