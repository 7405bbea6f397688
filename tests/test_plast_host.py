"""PlastDrift (tests/plastcases.py) on the host build of the device sources: the model against runs of the unmodified reference and
against the reference's known answer; od_plast_step against the reference's update_particle_depth + stokes_drift + advect_wind on
random inputs and against the helpers called one by one; the Philox stream of the analytical depths; the launches each path makes;
the configuration; and the refusal in distributed runs."""
import ctypes as C
import os
import socket
import sys
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import common
import plastcases as pc
import plast_host


@pytest.fixture()
def host_engine(monkeypatch):
    eng = plast_host.host_engine()
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    monkeypatch.setattr(E, 'default_engine', lambda device=None: eng)
    monkeypatch.setattr(B, 'default_engine', lambda device=None: eng)
    yield eng


def _expected_launches(case):
    """(od_plast_step, od_vertical_mixing) per run"""
    return pc.STEPS, (pc.STEPS if case in pc.RANDOMWALK else 0)


@pytest.mark.parametrize('case', list(pc.CASES))
def test_plast_case_equals_the_reference(case, host_engine):
    o = pc.run_product(case)
    pc.check(o, case)
    calls = host_engine.lib.calls
    plast, mix = _expected_launches(case)
    assert calls.count('od_plast_step') == plast
    assert calls.count('od_vertical_mixing') == mix
    if case != 'subclass_reference_update':
        assert calls.count('od_stokes_drift') == 0          # the Stokes move is inside od_plast_step


def test_the_cases_cover_what_they_name():
    ref = np.load(pc.GOLDEN)
    g = lambda case, k: ref['%s__%s' % (case, k)]        # noqa: E731
    assert not g('no_mixing', 'h_zf64').any() and g('analytical_tabularised', 'h_zf64').all()
    # the shallow floor: analytical depths below it after update(), lifted at the top of the next step
    fx = common.Fixture('rk4_3d_full')
    floor = pc.fields(fx)[4][0]
    assert g('shallow_floor', 'h_z').min() < -float(floor.max())
    assert 'seeded_on_land' in list(g('mask_previous', 'cats'))
    assert len(set(g('release_backward', 'h_len'))) > 1


def test_wind_drift_shear_known_answer(host_engine):
    """tests/models/test_models.py::test_wind_drift_shear of the reference, to its six decimals (the reference itself gives the same
    answer without the GSHHG landmask: tests/golden/plast_ref.npz, 'shear')"""
    from opendrift_b200.models.plastdrift import PlastDrift
    lon, lat = pc.run_shear(PlastDrift)
    np.testing.assert_array_almost_equal(lon, pc.SHEAR_LON)
    assert abs(lat[0] - lat[2]) < 0.5e-3
    ref = np.load(pc.GOLDEN)
    np.testing.assert_array_almost_equal(ref['shear__lon'], pc.SHEAR_LON)
    assert max(common.max_err_deg(lon, lat, ref['shear__lon'], ref['shear__lat'])) < pc.TOL_DEG


def test_configuration_follows_the_reference(host_engine):
    from opendrift_b200.models.plastdrift import PlastDrift, PlastElement
    o = PlastDrift(loglevel=50)
    assert o.get_config('vertical_mixing:mixingmodel') == 'analytical'
    assert o.get_config('drift:vertical_mixing') is True and o.get_config('drift:vertical_advection') is True
    assert o.get_config('drift:use_tabularised_stokes_drift') is True
    assert o.get_config('vertical_mixing:diffusivitymodel') == 'windspeed_Sundby1983'
    assert o.get_config('general:coastline_action') == 'none'
    assert PlastElement.variables['terminal_velocity']['default'] == 0.01
    assert PlastElement.variables['terminal_velocity']['dtype'] == np.float32
    from oracle import refrun
    refrun.setup()
    from opendrift.models.plastdrift import PlastDrift as RefPlast
    assert PlastDrift.required_variables == RefPlast.required_variables


# -- one launch against the reference's NumPy ------------------------------------------------------------------------------------------
def _random_inputs(n, rng, z_f64, tv_f64, wdf_f64):
    el = {'z': -rng.exponential(3.0, n), 'terminal_velocity': rng.uniform(0.001, 0.05, n),
          'wind_drift_factor': rng.uniform(0.0, 0.04, n), 'moving': (rng.uniform(0, 1, n) > 0.1).astype(np.int32)}
    el['z'][::11] = 0.0
    el['z'][1::11] = rng.uniform(0, 0.5, len(el['z'][1::11]))        # above the surface
    el['z'] = el['z'].astype(np.float64 if z_f64 else np.float32)
    el['terminal_velocity'] = el['terminal_velocity'].astype(np.float64 if tv_f64 else np.float32)
    el['wind_drift_factor'] = el['wind_drift_factor'].astype(np.float64 if wdf_f64 else np.float32)
    env = {k: rng.uniform(-15, 15, n).astype(np.float32) for k in ('x_wind', 'y_wind')}
    env['x_wind'][::17] = 0
    env['y_wind'][::17] = 0
    env['ocean_vertical_diffusivity'] = rng.uniform(0.0, 0.05, n).astype(np.float32)
    env['sea_surface_wave_stokes_drift_x_velocity'] = rng.uniform(-0.2, 0.2, n).astype(np.float32)
    env['sea_surface_wave_stokes_drift_y_velocity'] = rng.uniform(-0.2, 0.2, n).astype(np.float32)
    env['sea_surface_wave_significant_height'] = rng.uniform(0, 6, n).astype(np.float32)
    return el, env


def _special_scales(el, env):
    """K = 0, NaN K, tv = 0 (an infinite scale), tiny tv"""
    env['ocean_vertical_diffusivity'][::13] = 0.0
    env['ocean_vertical_diffusivity'][1::29] = np.nan
    el['terminal_velocity'][2::31] = 0.0
    el['terminal_velocity'][3::37] = 1e-30


class _Elements(types.SimpleNamespace):
    def __len__(self):
        return len(self.z)


def _reference_stub(el, env, cfg, moves):
    from oracle import refrun
    refrun.setup()
    from opendrift.models.plastdrift import PlastDrift as RefPlast
    from opendrift.models.physics_methods import PhysicsMethods
    n = len(el['z'])
    stub = types.SimpleNamespace(
        elements=_Elements(**{k: v.copy() for k, v in el.items()}),
        environment=types.SimpleNamespace(**{k: v.copy() for k, v in env.items()}),
        num_elements_active=lambda: n, update_positions=lambda u, v: moves.append((np.asarray(u), np.asarray(v))),
        get_config=lambda key, default=None: cfg.get(key, default))
    for name in ('stokes_drift', 'advect_wind', 'significant_wave_height', 'wave_period', '_wave_frequency', 'wind_speed'):
        setattr(stub, name, types.MethodType(getattr(PhysicsMethods, name), stub))
    stub.update_particle_depth = types.MethodType(RefPlast.update_particle_depth, stub)
    return stub


def _launch(eng, el, env, lon0, lat0, profile, wdd, seed, stokes=True):
    """od_plast_step on the host build from the same inputs, with the legacy generator seeded as the reference's was"""
    t = {k: torch.from_numpy(v.copy()) for k, v in env.items()}
    us, vs, hs = (t['sea_surface_wave_stokes_drift_x_velocity'], t['sea_surface_wave_stokes_drift_y_velocity'],
                  t['sea_surface_wave_significant_height'])
    hs_mode = 0 if env['sea_surface_wave_significant_height'].max() > 0 else 1
    lon, lat = torch.tensor(lon0), torch.tensor(lat0)
    n = len(lon0)
    np.random.seed(seed)
    draws = torch.from_numpy(np.random.standard_exponential(n))
    sub = (t['ocean_vertical_diffusivity'], torch.from_numpy(el['terminal_velocity'].copy()), draws,
           torch.arange(n, dtype=torch.int32), 0, 0)
    z = eng.plast_step(lon, lat, torch.from_numpy(el['moving'].copy()), torch.from_numpy(el['z'].copy()), 3600.0, submerge=sub,
                       stokes=(us, vs, hs, t['x_wind'], t['y_wind'], hs_mode, profile, None) if stokes else None,
                       wind=(t['x_wind'], t['y_wind'], torch.from_numpy(el['wind_drift_factor'].copy()), wdd))
    return lon.numpy(), lat.numpy(), z.numpy()


@pytest.mark.parametrize('profile', ['monochromatic', 'exponential', 'Phillips'])
@pytest.mark.parametrize('dtypes', [(False, False, False), (True, True, True), (True, False, True)])
@pytest.mark.parametrize('wdd', [0.1, 0.0, 3.0])
def test_plast_launch_equals_the_reference(profile, dtypes, wdd, host_engine):
    """The reference's update_particle_depth, stokes_drift and advect_wind on random elements, with the moves recorded instead of
    made, against one launch: the depths bit for bit, the positions after both moves (an hour) within 1e-9 degrees."""
    rng = np.random.default_rng(hash((profile, dtypes, wdd)) % 2**32)
    n = 4000
    el, env = _random_inputs(n, rng, *dtypes)
    _special_scales(el, env)
    lon0, lat0 = rng.uniform(-10, 10, n), rng.uniform(50, 70, n)
    cfg = {'drift:vertical_mixing': True, 'vertical_mixing:mixingmodel': 'analytical', 'drift:stokes_drift': True,
           'drift:stokes_drift_profile': profile, 'drift:wind_drift_depth': wdd, 'drift:relative_wind': False}
    moves = []
    stub = _reference_stub(el, env, cfg, moves)
    np.random.seed(5)
    with np.errstate(all='ignore'):
        stub.update_particle_depth()
        z_ref = stub.elements.z
        stub.stokes_drift()
        stub.advect_wind()
    eng = host_engine
    lon_e, lat_e = torch.tensor(lon0), torch.tensor(lat0)
    mv = torch.from_numpy(el['moving'].copy())
    for u, v in moves:
        eng.update_positions(lon_e, lat_e, torch.from_numpy(np.ascontiguousarray(u)), torch.from_numpy(np.ascontiguousarray(v)), mv,
                             3600.0)
    lon, lat, z = _launch(eng, el, env, lon0, lat0, profile, wdd, 5)
    assert z_ref.dtype == np.float64
    assert np.array_equal(z.view(np.int64)[~np.isnan(z)], z_ref.view(np.int64)[~np.isnan(z_ref)])
    assert np.array_equal(np.isnan(z), np.isnan(z_ref))
    assert np.isinf(z).any() and (z == 0).any() and np.isnan(z).any()
    # the wind move's dtype follows the reference's (float32 velocities when wind_drift_depth = 0 and wdf is float32)
    assert moves[-1][0].dtype == (np.float32 if wdd == 0 and not dtypes[2] else np.float64)
    # NaN and infinite depths give undefined Stokes velocities in both; compare where the depth is finite.  NumPy's float64 exp (SIMD)
    # against glibc's differ by an ulp here and there
    f = np.isfinite(z)
    err = max(common.max_err_deg(lon[f], lat[f], lon_e.numpy()[f], lat_e.numpy()[f]))
    assert err < 1e-9, err
    assert np.array_equal(np.isnan(lon), np.isnan(lon_e.numpy()))


@pytest.mark.parametrize('what', ['tv < 0', 'K = 0, tv < 0', 'tv = -0.0', 'K < 0'])
def test_negative_scale_raises_as_numpy_does(what, host_engine):
    rng = np.random.default_rng(9)
    n = 500
    el, env = _random_inputs(n, rng, False, False, False)
    k = 77
    if what == 'tv < 0':
        el['terminal_velocity'][k] = -0.01
    elif what == 'K = 0, tv < 0':
        env['ocean_vertical_diffusivity'][k] = 0.0
        el['terminal_velocity'][k] = -0.01
    elif what == 'tv = -0.0':
        el['terminal_velocity'][k] = -0.0
    else:
        env['ocean_vertical_diffusivity'][k] = -1e-3
    scale = env['ocean_vertical_diffusivity'] / el['terminal_velocity']
    with pytest.raises(ValueError, match='scale < 0') as ref_err:
        np.random.exponential(scale=scale, size=n)
    z0 = el['z'].copy()
    lon0, lat0 = rng.uniform(-10, 10, n), rng.uniform(50, 70, n)
    with pytest.raises(ValueError, match='scale < 0') as err:
        _launch(host_engine, el, env, lon0, lat0, 'Phillips', 0.1, 1)
    assert str(err.value) == str(ref_err.value)
    assert np.array_equal(el['z'], z0)
    # NaN scales pass (0 / 0 with the sign bit set)
    env['ocean_vertical_diffusivity'][k] = 0.0
    el['terminal_velocity'][k] = 0.0
    _launch(host_engine, el, env, lon0, lat0, 'Phillips', 0.1, 1)


def _helper_path(Model):
    """The same model with its stokes_drift wrapped: update() takes the helpers one by one (od_plast_step for the depth alone,
    od_stokes_drift, the advect_wind helper)."""
    class Helpers(Model):
        def stokes_drift(self, *a, **kw):
            return super().stokes_drift(*a, **kw)
    return Helpers


@pytest.mark.parametrize('case', ['analytical_tabularised', 'stokes_hs_readers', 'monochromatic', 'mixed_terminal_velocity',
                                  'randomwalk_environment', 'no_mixing', 'release_backward', 'uncertainty'])
def test_one_launch_equals_the_helpers_one_by_one(case, host_engine, monkeypatch):
    """Fusing update_particle_depth, stokes_drift and advect_wind into one launch changes no arithmetic: bit for bit."""
    from opendrift_b200.models import plastdrift
    fused = pc.summary(pc.run_product(case))
    monkeypatch.setattr(plastdrift, 'PlastDrift', _helper_path(plastdrift.PlastDrift))
    host_engine.lib.calls.clear()
    helpers = pc.summary(pc.run_product(case))
    assert host_engine.lib.calls.count('od_update_positions') >= pc.STEPS          # the advect_wind helper
    for k in fused:
        assert np.array_equal(fused[k], helpers[k], equal_nan=fused[k].dtype.kind == 'f'), k


# -- Philox -------------------------------------------------------------------------------------------------------------------------
def _philox_u0(n, seed, step, tag):
    s = plast_host.shim()
    ids = np.arange(n, dtype=np.int32)
    out = np.empty(n)
    assert s.hs6_philox_u0(n, seed, ids.ctypes.data_as(C.c_void_p), step, tag, out.ctypes.data_as(C.c_void_p)) == 0
    return out


def test_philox_depths_are_exponential_and_independent_of_the_mixing_stream(host_engine):
    """10^6 depths of the device generator with K / tv = 1: Exp(1) by a KS test, and uncorrelated with the mixing loop's first
    iteration (the same ID and step)."""
    import scipy.stats
    n = 1_000_000
    lon, lat = torch.zeros(n, dtype=torch.float64), torch.full((n,), 60.0, dtype=torch.float64)
    ones = torch.ones(n, dtype=torch.float32)
    z = host_engine.plast_step(lon, lat, None, torch.zeros(n, dtype=torch.float32), 3600.0,
                               submerge=(ones, ones, None, torch.arange(n, dtype=torch.int32), 1234, 3))
    e = -z.numpy()
    assert scipy.stats.kstest(e, 'expon').pvalue > 1e-3
    u_mix = _philox_u0(n, 1234, 3, 0)
    assert abs(np.corrcoef(1.0 - np.exp(-e), u_mix)[0, 1]) < 5e-3
    # the next step's draws are a different stream
    z2 = host_engine.plast_step(lon, lat, None, torch.zeros(n, dtype=torch.float32), 3600.0,
                                submerge=(ones, ones, None, torch.arange(n, dtype=torch.int32), 1234, 4))
    assert abs(np.corrcoef(e, -z2.numpy())[0, 1]) < 5e-3


# -- distributed runs --------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    sys.path.insert(0, common.ROOT)
    sys.path.insert(0, os.path.join(common.ROOT, 'tests'))
    import plast_host as ph
    import plastcases as cases
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    eng = ph.host_engine()
    E.default_engine = B.default_engine = lambda device=None: eng
    try:
        cases.run_product('no_mixing', extra_config={'gpu:rng': 'philox', 'drift:use_tabularised_stokes_drift': False})
        q.put((rank, 'ran', ''))
    except NotImplementedError as e:
        q.put((rank, 'refused', str(e)))
    dist.destroy_process_group()


def test_two_rank_run_refuses_the_model():
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in procs], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
    assert [r[1] for r in res] == ['refused', 'refused']
    assert all('PlastDrift' in r[2] for r in res)
