"""SedimentDrift (tests/sedimentcases.py) on the host build of the device sources: the model against runs of the unmodified
reference; od_resuspend against the reference's NumPy expressions restated here; the settling launch against the per-iteration
path with the Python bottom_interaction, bit for bit; the launches each path makes; the coastline default; and the refusal in
distributed runs."""
import logging
import os
import socket
import sys
from datetime import timedelta

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import common
import sedimentcases as sc
import sediment_host


@pytest.fixture()
def host_engine(monkeypatch):
    eng = sediment_host.host_engine()
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    monkeypatch.setattr(E, 'default_engine', lambda device=None: eng)
    monkeypatch.setattr(B, 'default_engine', lambda device=None: eng)
    yield eng


def _ntimes(case):
    return abs(sc.CASES[case][4]) // 60


@pytest.mark.parametrize('case', list(sc.CASES))
def test_sediment_case_equals_the_reference(case, host_engine):
    o = sc.run_product(case)
    sc.check(o, case)
    calls = host_engine.lib.calls
    assert calls.count('od_resuspend') == sc.STEPS
    if case == 'hook_subclass':            # a subclass's own bottom_interaction: one launch per inner iteration
        assert calls.count('od_vertical_mixing_settle') == 0
        assert calls.count('od_vertical_mixing') == sc.STEPS * _ntimes(case)
        assert o.n_hook > 0
    elif case == 'undecided_alone':        # undecided in every step: the step again on the per-iteration path
        assert calls.count('od_vertical_mixing_settle') == sc.STEPS
        assert calls.count('od_vertical_mixing') == sc.STEPS * _ntimes(case)
    elif case == 'undecided_sinker':       # undecided in the first step only: both elements have settled after it
        assert calls.count('od_vertical_mixing_settle') == sc.STEPS
        assert calls.count('od_vertical_mixing') == _ntimes(case)
    else:
        assert calls.count('od_vertical_mixing_settle') == sc.STEPS
        assert calls.count('od_vertical_mixing') == 0


def test_the_cases_cover_what_they_name():
    ref = np.load(sc.GOLDEN)
    g = lambda case, k: ref['%s__%s' % (case, k)]        # noqa: E731
    # settled elements, and elements that settled and were resuspended, in the history
    for case in ('example_fallback_floor', 'lift_profile', 'tidal_sundby'):
        assert (g(case, 'h_moving') == 0).sum() > 0 and (g(case, 'moving') == 1).sum() > 0
    # elements deactivated on the floor this step are resuspended too (moving = 1 in the removed elements)
    assert g('deactivate_profile', 'd_moving').sum() > 0 and len(g('deactivate_profile', 'd_id')) > 0
    # no reader for the floor: elements settle below the fallback depth
    z, mv = g('example_fallback_floor', 'z'), g('example_fallback_floor', 'moving')
    assert np.any(z[mv == 0] < -30)
    # a current of exactly float32(threshold): nothing is resuspended, though float64(float32(0.2)) > 0.2
    assert np.float64(np.float32(0.2)) > 0.2
    mv = g('speed_at_threshold_constant', 'h_moving').reshape(sc.STEPS, -1)
    assert np.all(mv[1:] <= mv[:-1]) and (mv[-1] == 0).sum() > 0
    # the constructed cases: element 0 settles with the sinker, never alone
    assert list(g('undecided_sinker', 'moving')) == [0, 0, 1, 1]
    assert list(g('undecided_alone', 'moving')) == [1, 1, 1, 1] and g('undecided_alone', 'z')[0] == -30.0


# -- od_resuspend against the reference's expressions ------------------------------------------------------------------------------
def _ref_resuspend(u, v, threshold, moving, z):
    """sedimentdrift.py:118-126 literally, on the float32 environment arrays (current_speed, physics_methods.py:889-891)."""
    moving, z = moving.copy(), z.copy()
    with np.errstate(invalid='ignore', over='ignore'):
        speed = np.sqrt(u ** 2 + v ** 2)
        resuspending = np.logical_and(speed > threshold, moving == 0)
    moving[resuspending] = 1
    z[resuspending] = z[resuspending] + .01
    return moving, z


def _resuspend_inputs(seed, n, threshold):
    rng = np.random.default_rng(seed)
    u = (rng.standard_normal(n) * 0.3).astype(np.float32)
    v = (rng.standard_normal(n) * 0.3).astype(np.float32)
    t32 = np.float32(threshold)
    special = [(np.nan, 0.0), (0.0, np.nan), (0.0, 0.0), (-0.0, -0.0), (t32, 0.0), (0.0, -t32), (-t32, 0.0),
               (np.nextafter(t32, np.float32(1)), 0.0), (np.nextafter(t32, np.float32(0)), 0.0), (np.inf, 0.0), (0.0, -np.inf),
               (np.inf, np.nan), (3e19, 3e19), (1e-30, 1e-30)]
    for k, (a, b) in enumerate(special[:n]):
        u[k], v[k] = a, b
    moving = (rng.random(n) < 0.5).astype(np.int32)
    moving[:len(special)] = 0
    z = -rng.random(n) * 50
    z[:3] = [0.0, -0.0, np.nan][:n]
    return u, v, moving, z


@pytest.mark.parametrize('threshold', [0.2, 0.5, 0.0, 3.0])
@pytest.mark.parametrize('z_dtype', [np.float32, np.float64])
def test_resuspend_equals_numpy(threshold, z_dtype):
    eng = sediment_host.host_engine()
    for seed in range(3):
        u, v, moving, z = _resuspend_inputs(seed, 5000, threshold)
        z = z.astype(z_dtype)
        want_m, want_z = _ref_resuspend(u, v, threshold, moving, z)
        dm, dz = torch.from_numpy(moving.copy()), torch.from_numpy(z.copy())
        eng.resuspend(torch.from_numpy(u), torch.from_numpy(v), threshold, dm, dz)
        assert np.array_equal(dm.numpy(), want_m)
        assert dz.dtype == torch.from_numpy(z).dtype
        assert np.array_equal(dz.numpy(), want_z, equal_nan=True) and np.array_equal(np.signbit(dz.numpy()), np.signbit(want_z))
    if threshold == 0.2:
        assert want_m[4] == 0 and want_m[5] == 0 and want_m[7] == 1       # exactly float32(0.2): not resuspended


# -- the settling launch against the per-iteration path ----------------------------------------------------------------------------
def run_scenario(seed, per_iteration=False, n=400, release=True, **kw):
    """A random SedimentDrift run: depths spread over the water column with some elements exactly on the floor, random terminal
    velocities (some 0), a random diffusivity model (some with K = 0) and sea-floor action.  per_iteration: the same model through
    a subclass whose bottom_interaction is SedimentDrift's, which takes the per-iteration path."""
    from opendrift_b200.models.sedimentdrift import SedimentDrift
    from opendrift_b200.readers import reader_regular_grid
    rng = np.random.default_rng(seed)
    fx = common.Fixture('rk4_3d_full')
    Model = SedimentDrift
    if per_iteration:
        class PerIteration(SedimentDrift):
            def bottom_interaction(self, seafloor_depth):
                SedimentDrift.bottom_interaction(self, seafloor_depth)
        Model = PerIteration
    np.random.seed(seed)
    o = Model(loglevel=50)
    floor_reader = bool(rng.random() < 0.6)
    floor_const = np.float32(rng.choice([20.0, 30.0, 35.5]))
    if floor_reader:
        floor, _, _, _, _ = sc.fields(fx)
        o.add_reader(reader_regular_grid.Reader(fx.grid_lon, fx.grid_lat, None, fx.times,
                                                {'sea_floor_depth_below_sea_level': np.repeat(floor[None], len(fx.times), axis=0)},
                                                name='floor'))
        o.set_config('general:seafloor_action', str(rng.choice(['none', 'lift_to_seafloor', 'deactivate'])))
    o.add_reader(reader_regular_grid.Reader(fx.grid_lon, fx.grid_lat, fx.grid_z, fx.times,
                                            {common.CUR[0]: fx.u, common.CUR[1]: fx.v}, name='current'))
    model = str(rng.choice(['constant', 'windspeed_Large1994', 'windspeed_Sundby1983']))
    cfg = dict(sc._BASE, **{'vertical_mixing:diffusivitymodel': model, 'environment:fallback:sea_floor_depth_below_sea_level': float(floor_const),
                            'environment:fallback:ocean_vertical_diffusivity': float(rng.choice([0.0, 0.0, 1e-3])),
                            'vertical_mixing:resuspension_threshold': float(rng.choice([0.1, 0.3])),
                            'drift:vertical_advection': False})
    cfg.update(kw)
    for k, val in cfg.items():
        o.set_config(k, val)
    z = (-rng.random(n) * 40).astype(np.float32)
    on_floor = rng.random(n) < 0.15
    z[on_floor] = -floor_const if not floor_reader else z[on_floor]
    tv = (-rng.random(n) * 0.01).astype(np.float32)
    tv[rng.random(n) < 0.3] = 0.0
    lon, lat = rng.uniform(2.3, 3.7, n), rng.uniform(56.2, 56.9, n)
    t = [fx.start, fx.start + timedelta(seconds=1800)] if release else fx.start
    o.seed_elements(lon=lon, lat=lat, z=z, time=t, terminal_velocity=tv)
    o.run(steps=5, time_step=900, time_step_output=900)
    return o


def _same(a, b):
    """The same elements with the same values, bit for bit, compared by ID (with the device generator the arrays are sorted by cell,
    and elements of one cell land in the order the sort's atomic counters give them)."""
    for ea, eb, keys in ((a.elements, b.elements, ('ID', 'lon', 'lat', 'z', 'moving', 'status')),
                         (a.elements_deactivated, b.elements_deactivated, ('ID', 'z', 'moving', 'status'))):
        ia, ib = np.argsort(np.asarray(ea.ID)), np.argsort(np.asarray(eb.ID))
        for k in keys:
            x, y = np.asarray(getattr(ea, k)), np.asarray(getattr(eb, k))
            assert x.dtype == y.dtype and np.array_equal(x[ia], y[ib], equal_nan=True), k
    assert list(a.status_categories) == list(b.status_categories)


@pytest.mark.parametrize('rng_kind', ['numpy', 'philox'])
@pytest.mark.parametrize('seed', range(8))
def test_settling_launch_equals_the_per_iteration_path(seed, rng_kind, host_engine):
    a = run_scenario(seed, **{'gpu:rng': rng_kind})
    calls = list(host_engine.lib.calls)
    host_engine.lib.calls.clear()
    b = run_scenario(seed, per_iteration=True, **{'gpu:rng': rng_kind})
    assert host_engine.lib.calls.count('od_vertical_mixing_settle') == 0
    _same(a, b)
    assert calls.count('od_vertical_mixing_settle') == 5


def test_the_scenarios_have_undecided_steps_and_steps_without(host_engine):
    """Among the random scenarios, some steps were redone (elements on the floor with K = 0 and w = 0) and some were not."""
    redone, clean = 0, 0
    for seed in range(8):
        host_engine.lib.calls.clear()
        run_scenario(seed)
        c = host_engine.lib.calls
        if c.count('od_vertical_mixing'):
            redone += 1
        else:
            clean += 1
    assert redone > 0 and clean > 0, (redone, clean)


# -- coastline default -------------------------------------------------------------------------------------------------------------
def test_coastline_warning_names_the_reference_default_of_the_model(host_engine, caplog):
    from opendrift_b200.models.oceandrift import OceanDrift
    from opendrift_b200.models.sedimentdrift import SedimentDrift
    from opendrift_b200.readers import reader_regular_grid
    fx = common.Fixture('rk4_3d_full')
    _, _, _, _, mask = sc.fields(fx)
    msgs = {}
    for Model in (OceanDrift, SedimentDrift):
        o = Model(loglevel=50)
        assert o.get_config('general:coastline_action') == 'none'
        o.add_reader(reader_regular_grid.Reader(fx.grid_lon, fx.grid_lat, None, fx.times,
                                                {'land_binary_mask': np.repeat(mask[None], len(fx.times), axis=0)}, name='mask'))
        o.set_config('general:use_auto_landmask', False)
        o.seed_elements(lon=fx.lon0[:20], lat=fx.lat0[:20], time=fx.start)
        caplog.clear()
        with caplog.at_level(logging.WARNING):
            o.run(steps=1, time_step=900)
        msgs[Model.__name__] = [r.getMessage() for r in caplog.records if 'land_binary_mask' in r.getMessage()]
    assert msgs['OceanDrift'] == [
        "a reader provides land_binary_mask but general:coastline_action is 'none' (the default of the GPU classes; the "
        "reference's default is 'stranding'): set general:coastline_action = 'stranding' and "
        "general:coastline_approximation_precision = None to strand elements on that mask"]
    assert len(msgs['SedimentDrift']) == 1 and "reference's default is 'previous'" in msgs['SedimentDrift'][0]
    assert "general:coastline_action = 'previous'" in msgs['SedimentDrift'][0]


def test_model_defaults():
    from opendrift_b200.models.sedimentdrift import SedimentDrift, SedimentElement
    o = SedimentDrift(loglevel=50)
    assert o.get_config('drift:vertical_mixing') is True
    assert o.get_config('vertical_mixing:resuspension_threshold') == 0.2
    assert SedimentElement.variables['settled']['dtype'] is np.uint8
    assert SedimentElement.variables['terminal_velocity']['default'] == -0.001
    assert o.required_variables['ocean_vertical_diffusivity'] == {'fallback': 0.02, 'profiles': True}


def test_seafloor_previous_with_mixing_is_refused(host_engine):
    from opendrift_b200.models.sedimentdrift import SedimentDrift
    from opendrift_b200.readers import reader_regular_grid
    fx = common.Fixture('rk4_3d_full')
    floor, _, _, _, _ = sc.fields(fx)
    o = SedimentDrift(loglevel=50)
    o.add_reader(reader_regular_grid.Reader(fx.grid_lon, fx.grid_lat, None, fx.times,
                                            {'sea_floor_depth_below_sea_level': np.repeat(floor[None], len(fx.times), axis=0)}, name='floor'))
    for k, v in dict(sc._BASE, **{'general:seafloor_action': 'previous'}).items():
        o.set_config(k, v)
    o.seed_elements(lon=fx.lon0[:20], lat=fx.lat0[:20], z=-5.0, time=fx.start)
    with pytest.raises(NotImplementedError, match="seafloor_action = 'previous'"):
        o.run(steps=1, time_step=900)


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
    import sediment_host as sh
    import sedimentcases as cases
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    eng = sh.host_engine()
    E.default_engine = B.default_engine = lambda device=None: eng
    try:
        cases.run_product('lift_profile', extra_config={'gpu:rng': 'philox'})
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
    assert all('SedimentDrift' in r[2] for r in res)
