"""LarvalFish (tests/larvalcases.py) on the host build of the device sources: the model against runs of the unmodified reference; od_larval_develop and od_larval_migrate against the reference's update_fish_larvae, update_terminal_velocity and
larvae_vertical_migration on random inputs; the fused step against the helpers called one by one; the launches each path makes;
the configuration; and the refusal in distributed runs."""
import os
import socket
import sys
import types
from datetime import datetime, timedelta

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import common
import larvalcases as lc
import larval_host


@pytest.fixture()
def host_engine(monkeypatch):
    eng = larval_host.host_engine()
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    monkeypatch.setattr(E, 'default_engine', lambda device=None: eng)
    monkeypatch.setattr(B, 'default_engine', lambda device=None: eng)
    yield eng


def _steps(case):
    ref = np.load(lc.GOLDEN)
    return len(ref['%s__h_len' % case])


@pytest.mark.parametrize('case', list(lc.CASES) + [lc.EXAMPLE])
def test_larval_case_equals_the_reference(case, host_engine):
    o, err = lc.run_product(case)
    lc.check(o, case, err)
    calls = host_engine.lib.calls
    steps = _steps(case)
    mixing = case == lc.EXAMPLE or lc.CASES[case][0].get('drift:vertical_mixing', True)
    if case in lc.RAISES:
        assert isinstance(err, ValueError) and calls.count('od_larval_develop') == 1
        return
    assert calls.count('od_larval_develop') == steps * (2 if case == 'subclass_reference_update' else 1)
    assert calls.count('od_larval_migrate') == steps
    assert calls.count('od_vertical_mixing') == (steps if mixing else 0)


def test_the_raises_are_the_references():
    ref = np.load(lc.GOLDEN)
    assert str(ref['hot_temperature__error']) == 'ValueError' and str(ref['no_eggs_no_larvae__error']) == 'ValueError'
    # the temperature check comes after the current move (the positions moved, the terminal velocity is the seeded default) ...
    fx = common.Fixture('rk4_3d_full')
    assert not np.array_equal(ref['hot_temperature__lon'], np.resize(fx.lon0, lc.N).astype(np.float64))
    assert str(ref['hot_temperature__terminal_velocity_dtype']) == 'float64'
    assert (ref['hot_temperature__hatched'] == 1).sum() > lc.N // 2      # hatching came before it
    # ... the empty eggs' max before it
    np.testing.assert_array_equal(ref['no_eggs_no_larvae__lon'], np.resize(fx.lon0, lc.N).astype(np.float32))


def test_the_cases_cover_what_they_name():
    ref = np.load(lc.GOLDEN)
    g = lambda case, k: ref['%s__%s' % (case, k)]        # noqa: E731
    assert list(g('default_scalar', 'h_z_dtype'))[-1] == 'float64' and list(g('no_mixing', 'h_z_dtype')) == ['float32'] * lc.STEPS
    h0 = g('ts_arrays_hatching', 'h_hatched')[:lc.N]
    assert (g('ts_arrays_hatching', 'hatched') == 1).sum() > (h0 == 1).sum()           # eggs hatched during the run
    assert not np.array_equal(g('swim_0', 'z'), g('swim_1', 'z'))
    assert 'seafloor' in list(g('floor_deactivate', 'cats')) and 'stranded' in list(g('mask_stranding', 'cats'))
    assert len(set(g('release_backward', 'h_len'))) > 1
    # the example: the default (scalar, so float64) hatched, weight and length, and larvae that grow and swim
    ex = lambda k: g(lc.EXAMPLE, k)                      # noqa: E731
    assert [str(ex(v + '_dtype')) for v in lc.VARS] == ['float64'] * 6
    assert (ex('hatched') == 1).all() and (ex('weight') > 0.08).all() and (ex('length') > 0).all()
    assert (ex('h_hatched') == 0).any()


def test_configuration_follows_the_reference(host_engine):
    from opendrift_b200.models.larvalfish import LarvalFish, LarvalFishElement
    from oracle import refrun
    refrun.setup()
    from opendrift.models.larvalfish import LarvalFish as RefLarval, LarvalFishElement as RefElement
    o = LarvalFish(loglevel=50)
    assert o.get_config('IBM:fraction_of_timestep_swimming') == 0.15
    spec = o._config['IBM:fraction_of_timestep_swimming']
    assert (spec['min'], spec['max']) == (0.0, 1.0)
    for k in ('drift:vertical_mixing', 'drift:vertical_mixing_at_surface', 'drift:vertical_advection_at_surface'):
        assert o.get_config(k) is True
    assert o.get_config('general:coastline_action') == 'none'
    assert LarvalFish.required_variables == RefLarval.required_variables
    for v, spec in RefElement.variables.items():
        assert LarvalFishElement.variables[v]['dtype'] == spec['dtype'] and LarvalFishElement.variables[v].get('default') == spec.get('default')


def test_numpy_helpers_are_the_references():
    from opendrift_b200.models.physics_methods import PhysicsMethods, seawater_dynamic_viscosity
    from opendrift_b200.models.larvalfish import LarvalFish
    from oracle import refrun
    refrun.setup()
    from opendrift.models import physics_methods as rp
    from opendrift.models.larvalfish import LarvalFish as RefLarval
    rng = np.random.default_rng(5)
    for dt in (np.float32, np.float64):
        t, s = rng.uniform(-2, 30, 1000).astype(dt), rng.uniform(0, 40, 1000).astype(dt)
        np.testing.assert_array_equal(PhysicsMethods.sea_water_density(t, s), rp.PhysicsMethods.sea_water_density(t, s))
        for m in ('sharqawy', 'ladim'):
            np.testing.assert_array_equal(seawater_dynamic_viscosity(t, s, m), rp.seawater_dynamic_viscosity(t, s, m))
        w = rng.uniform(0.01, 5, 1000).astype(dt)
        me = types.SimpleNamespace(time_step=timedelta(seconds=900))
        np.testing.assert_array_equal(LarvalFish.fish_growth(me, w, t.astype(np.float32)), RefLarval.fish_growth(me, w, t.astype(np.float32)))
    with pytest.raises(ValueError, match='celcius'):
        PhysicsMethods.sea_water_density(np.array([10, 100.5], np.float32), 35)


# -- the launches against the reference's NumPy on random inputs -------------------------------------------------------------------
def _random_elements(n, rng, f64):
    """Element arrays in the dtypes f64 names (a set of variable names seeded as scalars, i.e. float64), with the edge cases."""
    el = {'hatched': rng.integers(0, 2, n).astype(np.float64 if 'hatched' in f64 else np.uint8),
          'stage_fraction': rng.uniform(0.5, 1.0, n), 'weight': rng.uniform(0.01, 3, n), 'length': rng.uniform(3, 20, n),
          'diameter': rng.uniform(0.0003, 0.002, n), 'neutral_buoyancy_salinity': rng.uniform(29, 37, n), 'z': -rng.uniform(0, 40, n)}
    el['hatched'][::23] = 2                            # neither egg nor larva
    el['weight'][1::29] = 0.0                          # log(0) = -inf
    el['weight'][2::31] = -0.5                         # NaN
    el['length'][3::37] = 0.0                          # an infinite swimming speed
    el['z'][4::19] = 0.0
    el['z'][5::41] = -0.0
    for v in el:
        if v != 'hatched':
            el[v] = el[v].astype(np.float64 if v in f64 else np.float32)
    return el


def _random_environment(n, rng):
    t = rng.uniform(-2, 25, n).astype(np.float32)
    s = rng.uniform(25, 38, n).astype(np.float32)
    t[::17] = np.nan
    t[1::43] = 0.0
    t[2::47] = -0.0
    return t, s


def _edge_cases(el, t, s, dt):
    """A stage fraction that lands exactly on 1, and diameters on both sides of the 0.5 Reynolds limit."""
    # stage_fraction + days / exp(3.65 - 0.145 T) == 1 exactly in float32 for T = 10 (float64 when stage_fraction is)
    f32 = el['stage_fraction'].dtype == np.float32
    c = np.float32
    frac = c(dt / 86400) / np.exp(c(3.65) - c(0.145) * c(10.0))
    for k in range(6, len(t), 53):
        t[k] = 10.0
        el['hatched'][k] = 0
        el['stage_fraction'][k] = (c(1.0) - frac) if f32 else (1.0 - np.float64(frac))
    # dr = 0: the egg's salinity is the water's
    el['neutral_buoyancy_salinity'][7::59] = s[7::59]


class _Ref(types.SimpleNamespace):
    """The attributes the reference's LarvalFish methods read, over host arrays."""


def _reference(el, t, s, dt, hour, fraction):
    """The reference's update_fish_larvae, update_terminal_velocity and larvae_vertical_migration on copies (in that order, as in
    update()).  Returns (the arrays after each, or the exception raised)."""
    from oracle import refrun
    refrun.setup()
    from opendrift.models.larvalfish import LarvalFish as R
    from opendrift.models.physics_methods import PhysicsMethods as RP
    els = types.SimpleNamespace(**{k: v.copy() for k, v in el.items()})
    els.terminal_velocity = np.zeros(len(t), np.float32)
    me = _Ref(elements=els, environment=types.SimpleNamespace(sea_water_temperature=t.copy(), sea_water_salinity=s.copy()),
              time_step=timedelta(seconds=dt), time=datetime(2024, 3, 1, hour), sea_water_density=RP.sea_water_density,
              get_config=lambda k: fraction)
    me.fish_growth = types.MethodType(R.fish_growth, me)
    out = {}
    for name in ('update_fish_larvae', 'update_terminal_velocity', 'larvae_vertical_migration'):
        with np.errstate(all='ignore'):
            getattr(R, name)(me)
    for k in ('hatched', 'stage_fraction', 'weight', 'length', 'terminal_velocity', 'z'):
        out[k] = getattr(els, k)
    return out


def _launch(eng, el, t, s, dt, hour, fraction, dev=torch.device('cpu')):
    """The two launches as LarvalFish runs them: develop with the terminal velocity, then the migration."""
    d = {k: torch.from_numpy(v.copy()).to(dev) for k, v in el.items()}
    w, flags = eng.larval_develop(torch.from_numpy(t.copy()).to(dev), torch.from_numpy(s.copy()).to(dev), d, dt)
    eng.larval_migrate(d['hatched'], d['length'], d['z'], fraction, -1 if hour < 12 else 1, dt)
    out = {k: v.cpu().numpy() for k, v in d.items()}
    out['terminal_velocity'] = w.cpu().numpy()
    return out, flags


def _ulps(a, b):
    """the largest difference in float32 ulps of b where both are finite: every chain starts from the float32 temperature, so a
    float64 result carries float32 roundings too"""
    f = np.isfinite(a) & np.isfinite(b)
    if not f.any():
        return 0.0
    sp = np.spacing(np.abs(b[f]).astype(np.float32)).astype(np.float64)
    return float(np.max(np.abs(a[f].astype(np.float64) - b[f]) / sp))


DTYPE_FLOWS = [(), ('hatched',), ('stage_fraction', 'weight'), ('length',), ('diameter',), ('neutral_buoyancy_salinity',), ('z',),
               ('weight', 'length', 'diameter', 'neutral_buoyancy_salinity', 'z', 'hatched', 'stage_fraction')]
# bounds on the differences from the reference over these inputs, in float32 ulps of each output (largest seen: stage_fraction 1,
# weight 2, length 5, terminal_velocity 6, z 45).  NumPy's float32 exp / log / log10 / pow are SIMD routines (up to 2-3 ulp), the
# launches use the float64 functions rounded to float32; the growth and the terminal velocity chain several of them, the density
# difference dr cancels, and the migration adds a swimming distance whose terms 0.261 L^(1.552 L^-0.08) and 5.289 / L cancel.
ULP_BOUND = {'stage_fraction': 2, 'weight': 4, 'length': 8, 'terminal_velocity': 16, 'z': 64}


@pytest.mark.parametrize('f64', DTYPE_FLOWS, ids=lambda f: '+'.join(f) or 'float32')
@pytest.mark.parametrize('dt,hour', [(3600.0, 3), (-900.0, 15)])
def test_launches_equal_the_reference(f64, dt, hour, host_engine):
    rng = np.random.default_rng(len(f64) + abs(int(dt)))
    n = 5000
    el = _random_elements(n, rng, set(f64))
    t, s = _random_environment(n, rng)
    _edge_cases(el, t, s, dt)
    ref = _reference(el, t, s, dt, hour, 0.4)
    got, flags = _launch(host_engine, el, t, s, dt, hour, 0.4)
    assert flags & host_engine.LARVAL_STAGED and flags & host_engine.LARVAL_NAN_T and not flags & host_engine.LARVAL_HOT
    np.testing.assert_array_equal(got['hatched'], ref['hatched'])
    worst = {}
    for k in ULP_BOUND:
        a, b = got[k], ref[k]
        assert a.dtype == b.dtype, (k, a.dtype, b.dtype)
        assert np.array_equal(np.isnan(a), np.isnan(b)), k
        assert np.array_equal(np.isinf(a), np.isinf(b)) and np.array_equal(a[np.isinf(a)], b[np.isinf(b)]), k
        worst[k] = _ulps(a, b)
        assert worst[k] <= ULP_BOUND[k], (k, worst[k])
    print('largest ulp differences', worst)


def test_the_flags_raise_as_the_reference_does(host_engine):
    rng = np.random.default_rng(9)
    n = 300
    el = _random_elements(n, rng, set())
    t, s = _random_environment(n, rng)
    t[~np.isfinite(t)] = 5.0
    t[10] = 100.5
    _, flags = _launch(host_engine, el, t, s, 900.0, 3, 0.15)
    assert flags & host_engine.LARVAL_HOT and not flags & host_engine.LARVAL_NAN_T
    with pytest.raises(ValueError, match='celcius'):
        _reference(el, t, s, 900.0, 3, 0.15)
    t[11] = np.nan                                      # np.max is NaN: no raise
    _reference(el, t, s, 900.0, 3, 0.15)
    _, flags = _launch(host_engine, el, t, s, 900.0, 3, 0.15)
    assert flags & host_engine.LARVAL_HOT and flags & host_engine.LARVAL_NAN_T
    el['hatched'][:] = 2
    _, flags = _launch(host_engine, el, t, s, 900.0, 3, 0.15)
    assert not flags & host_engine.LARVAL_STAGED
    with pytest.raises(ValueError, match='zero-size'):
        _reference(el, t, s, 900.0, 3, 0.15)


# -- the fused step against the helpers --------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', ['ts_arrays_hatching', 'default_scalar', 'noon_crossing', 'floor_deactivate'])
@pytest.mark.parametrize('hook', ['larvae_vertical_migration', 'update_fish_larvae'])
def test_fused_step_equals_the_helpers_one_by_one(case, hook, host_engine, monkeypatch):
    from opendrift_b200.models.larvalfish import LarvalFish
    a = lc.summary(*lc.run_product(case))
    n_fused = host_engine.lib.calls.count('od_larval_develop')
    base = getattr(LarvalFish, hook)
    # an override that does what LarvalFish does
    Sub = type('Sub', (LarvalFish,), {hook: lambda self, *args: base(self, *args)})
    b = lc.summary(*lc.run_product(case, model=Sub))
    assert host_engine.lib.calls.count('od_larval_develop') - n_fused == 2 * n_fused
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_an_own_terminal_velocity_takes_the_per_iteration_path(host_engine, monkeypatch):
    from opendrift_b200.models.larvalfish import LarvalFish
    base = LarvalFish.update_terminal_velocity
    Sub = type('Sub', (LarvalFish,), {'update_terminal_velocity': lambda self, *a, **kw: base(self, *a, **kw)})
    o, _ = lc.run_product('ts_arrays_hatching', model=Sub)
    lc.check(o, 'ts_arrays_hatching')
    calls = host_engine.lib.calls
    assert calls.count('od_vertical_mixing') == lc.STEPS * 15          # one launch per inner iteration


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
    import larval_host as lh
    import larvalcases as cases
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    eng = lh.host_engine()
    E.default_engine = B.default_engine = lambda device=None: eng
    try:
        cases.run_product('no_mixing', extra_config={'gpu:rng': 'philox'})
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
    assert all('LarvalFish' in r[2] for r in res)
