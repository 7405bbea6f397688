"""ShipDrift (tests/shipcases.py) on the host build of the device sources: the model against runs of the unmodified reference; the
wave force table lookup against scipy's LinearNDInterpolator, bit for bit; the per-ship launch against the reference's update() on
random inputs; the launches per step; and the refusal in distributed runs."""
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
import shipcases as sc
import shipdrift_host


@pytest.fixture()
def host_engine(monkeypatch):
    eng = shipdrift_host.host_engine()
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    monkeypatch.setattr(E, 'default_engine', lambda device=None: eng)
    monkeypatch.setattr(B, 'default_engine', lambda device=None: eng)
    yield eng


@pytest.mark.parametrize('case', list(sc.CASES))
def test_ship_case_equals_the_reference(case, host_engine):
    o = sc.run_product(case)
    err = sc.check(o, case)
    print('%s: max position difference %.2e deg' % (case, err))
    # one launch per step; a subclass's own update() runs on the helper path instead
    assert host_engine.lib.calls.count('od_ship_step') == (0 if case == 'subclass_reference_update' else sc.STEPS)


def test_the_cases_cover_what_they_name():
    ref = np.load(sc.GOLDEN)
    g = lambda case, k: ref['%s__%s' % (case, k)]        # noqa: E731
    assert 'ship stranded' in list(g('mask_none', 'cats')) and len(g('mask_none', 'd_id')) > 0
    assert 'stranded' in list(g('mask_stranding', 'cats')) and 'ship stranded' not in list(g('mask_stranding', 'cats'))
    assert 'missing_data' in list(g('missing_wind', 'cats')) and len(g('missing_wind', 'd_id')) > 0
    assert len(set(g('release_backward', 'h_len'))) > 1


def _table():
    from opendrift_b200.models import shipdrift as sd
    wf = sd.read_wforce(sc.wforce_path())
    ipF, ipD = sd.wforce_interpolators(wf)
    return wf, ipF, ipD, sd.wforce_table(wf, ipF)


def test_wforce_lookup_is_scipys_bit_for_bit():
    wf, ipF, ipD, (wtab, wbox, dims) = _table()
    s = shipdrift_host.shim()
    dom = (12.0 - 2.25) / 99
    # the 49 frequencies the reference queries (the first, 2.25, lies on the table's outer face; none lies on an inner omega face,
    # where scipy's walk and the first tetrahedron of the box may take different neighbours and differ in the last bit)
    omegas = [2.25 + i * dom for i in range(100) if 2.25 + i * dom < 7.0]
    assert omegas[0] == wf['omega'][0] and not set(omegas[1:]) & set(wf['omega'])
    rng = np.random.default_rng(11)
    n = 400
    bl = np.clip(np.clip(rng.uniform(0.1, 0.2, n).astype(np.float32), 0.12, 0.18), 0.121, 0.179)
    dl = np.clip(np.clip(rng.uniform(0.02, 0.08, n).astype(np.float32), 0.025, 0.07), 0.0251, 0.069)
    bl[:40] = np.float32(0.121)            # the clip limits, and grid values of the table inside them
    bl[40:80] = np.float32(0.179)
    bl[80:100] = 0.14
    dl[::5] = np.float32(0.0251)
    dl[1::5] = np.float32(0.069)
    dl[2::9] = 0.055
    for om in omegas:
        # the reference calls the interpolator with one omega and the arrays of all elements
        f_ref, d_ref = ipF(om, bl, dl), ipD(om, bl, dl)
        o64, b64, d64 = np.full(n, om), bl.astype(np.float64), dl.astype(np.float64)
        f, d = np.empty(n), np.empty(n)
        ptr = lambda a: a.ctypes.data_as(C.c_void_p)        # noqa: E731
        assert s.hs5_ship_wforce(n, ptr(o64), ptr(b64), ptr(d64), ptr(wtab), ptr(wbox), *dims, ptr(f), ptr(d)) == 0
        assert np.array_equal(f.view(np.int64), f_ref.view(np.int64)), om
        assert np.array_equal(d.view(np.int64), d_ref.view(np.int64)), om


def _reference_update():
    from oracle import refrun
    refrun.setup()
    from opendrift.models.shipdrift import ShipDrift as RefShip
    from opendrift.models.physics_methods import PhysicsMethods
    return RefShip, PhysicsMethods


def _random_inputs(n, rng, period):
    """float32 element and environment arrays; ws = 0 for some ships, periods of exactly 5.7 and 8.55 s for others"""
    el = {'length': rng.uniform(20, 300, n), 'height': None, 'draft': None, 'beam': None}
    el['length'] = el['length'].astype(np.float32)
    el['beam'] = (el['length'] * rng.uniform(0.1, 0.2, n)).astype(np.float32)
    el['draft'] = (el['length'] * rng.uniform(0.02, 0.08, n)).astype(np.float32)
    el['height'] = (el['draft'] + rng.uniform(2, 50, n)).astype(np.float32)
    el['wind_drag_coeff'] = rng.uniform(0.7, 1.4, n).astype(np.float32)
    el['water_drag_coeff'] = rng.uniform(1.27, 1.5, n).astype(np.float32)
    el['orientation'] = (np.arange(n) % 2).astype(np.uint8)
    env = {k: rng.uniform(-15, 15, n).astype(np.float32) for k in ('x_wind', 'y_wind')}
    env['x_wind'][::17] = 0
    env['y_wind'][::17] = 0
    env.update({k: rng.uniform(-0.5, 0.5, n).astype(np.float32) for k in common.CUR})
    env['sea_surface_wave_significant_height'] = rng.uniform(0, 6, n).astype(np.float32) if period != 'wind' else np.zeros(n, np.float32)
    T = rng.uniform(2, 14, n).astype(np.float32) if period != 'wind' else np.zeros(n, np.float32)
    if period == 'reader':
        T[::7] = np.float32(5.7)
        T[1::7] = np.float32(8.55)
    if period == 'partial':
        T[::3] = 0
    env[sc.TM02] = T
    env['sea_surface_wave_stokes_drift_x_velocity'] = rng.uniform(-0.2, 0.2, n).astype(np.float32)
    env['sea_surface_wave_stokes_drift_y_velocity'] = rng.uniform(-0.2, 0.2, n).astype(np.float32)
    env['land_binary_mask'] = (rng.uniform(0, 1, n) < 0.1).astype(np.float32)
    return el, env


@pytest.mark.parametrize('period', ['wind', 'reader', 'partial'])
@pytest.mark.parametrize('stokes', [False, True])
def test_ship_launch_equals_the_reference_update(period, stokes, host_engine):
    """The reference's update() on random ships, with the moves recorded instead of made, against one launch: the positions after
    both moves, an hour later, within 1e-5 of the distance travelled."""
    RefShip, PM = _reference_update()
    rng = np.random.default_rng(3 if stokes else 4)
    n = 3000
    el, env = _random_inputs(n, rng, period)
    if not stokes:
        env['sea_surface_wave_stokes_drift_x_velocity'][:] = 0
        env['sea_surface_wave_stokes_drift_y_velocity'][:] = 0
    wf, ipF, ipD, table = _table()
    lon0 = rng.uniform(-10, 10, n)
    lat0 = rng.uniform(50, 70, n)
    moves, deact = [], []
    stub = types.SimpleNamespace(
        elements=types.SimpleNamespace(**{k: v.copy() for k, v in el.items()}),
        environment=types.SimpleNamespace(**{k: v.copy() for k, v in env.items()}),
        wforce_interpolator_F=ipF, wforce_interpolator_D=ipD, winwav_angle=RefShip.winwav_angle,
        num_elements_active=lambda: n, update_positions=lambda u, v: moves.append((np.asarray(u), np.asarray(v))),
        deactivate_elements=lambda idx, reason: deact.append((np.asarray(idx).copy(), reason)))
    for name in ('wave_period', 'significant_wave_height', '_wave_frequency', 'wind_speed'):
        setattr(stub, name, types.MethodType(getattr(PM, name), stub))
    RefShip.update(stub)
    # the expected positions: the recorded velocities through the same moves (od_update_positions of the host build)
    eng = host_engine
    lon_e, lat_e = torch.tensor(lon0), torch.tensor(lat0)
    mv = torch.ones(n, dtype=torch.int32)
    for u, v in moves:
        eng.update_positions(lon_e, lat_e, torch.from_numpy(u.copy()), torch.from_numpy(v.copy()), mv, 3600.0)
    assert moves[0][0].dtype == np.float32 and moves[1][0].dtype == np.float64
    # one launch, with the host's decisions taken as ShipDrift.update takes them
    T = env[sc.TM02]
    tm_wind = not T.max() > 0
    fill = np.mean(T[T > 0]) if not tm_wind and T.min() == 0 else None
    hs_wind = not env['sea_surface_wave_significant_height'].max() > 0
    t = {k: torch.from_numpy(v.copy()) for k, v in env.items()}
    envd = {'x_sea_water_velocity': t[common.CUR[0]], 'y_sea_water_velocity': t[common.CUR[1]], 'x_wind': t['x_wind'],
            'y_wind': t['y_wind'], 'hs': t['sea_surface_wave_significant_height'], 'period': t[sc.TM02],
            'stokes_x': t['sea_surface_wave_stokes_drift_x_velocity'] if stokes else None,
            'stokes_y': t['sea_surface_wave_stokes_drift_y_velocity'] if stokes else None, 'land_binary_mask': t['land_binary_mask']}
    lon, lat = torch.tensor(lon0), torch.tensor(lat0)
    status, moving = torch.zeros(n, dtype=torch.int32), torch.ones(n, dtype=torch.int32)
    eld = {k: torch.from_numpy(el[k].copy()) for k in ('length', 'height', 'draft', 'beam', 'wind_drag_coeff', 'water_drag_coeff')}
    tab = tuple(torch.from_numpy(a) for a in table[:2]) + (table[2],)
    stranded = eng.ship_step(lon, lat, moving, status, eld, torch.from_numpy(el['orientation'].copy()), envd, tab, 3600.0,
                             hs_wind=hs_wind, tm_wind=tm_wind, tm_fill=fill, strand_code=3)
    # NumPy's float32 exp / power (SIMD, 1 - 2.3 ulp) against the rounded float64 functions: the ship moves differ by up to a few
    # 1e-6 of the distance travelled, about 3 cm after an hour
    err_m = np.hypot((lon.numpy() - lon_e.numpy()) * np.cos(np.radians(lat0)) * 111320.0, (lat.numpy() - lat_e.numpy()) * 110574.0)
    travelled = np.hypot(moves[1][0], moves[1][1]) * 3600.0
    assert np.max(err_m / np.maximum(travelled, 1.0)) < 1e-5, (np.max(err_m / np.maximum(travelled, 1.0)), err_m.max())
    # Hs and the period written back into the environment as the reference writes them
    if hs_wind:
        assert np.array_equal(envd['hs'].numpy(), stub.environment.sea_surface_wave_significant_height)
    if tm_wind:
        assert np.array_equal(envd['period'].numpy(), getattr(stub.environment, sc.TM02).astype(np.float32))   # (a recarray field)
    idx, reason = deact[0]
    assert reason == 'ship stranded' and stranded == bool(idx.any())
    assert np.array_equal(status.numpy() == 3, idx) and np.array_equal(moving.numpy() == 0, idx)


def test_missing_table_names_the_keyword(monkeypatch):
    from opendrift_b200.models import shipdrift as sd
    monkeypatch.setattr(sd, 'find_wforce', lambda: None)
    with pytest.raises(FileNotFoundError, match='wforce='):
        sd.ShipDrift()


def test_seed_reproduces_the_reference_coefficients(host_engine):
    RefShip, _ = _reference_update()
    from opendrift_b200.models.shipdrift import ShipDrift
    kw = sc.sizes('mixed', 50)
    ours = ShipDrift(wforce=sc.wforce_path(), loglevel=50)
    ref = RefShip(loglevel=50)
    for o in (ours, ref):
        for v in ('x_wind', 'y_wind', 'x_sea_water_velocity', 'y_sea_water_velocity', 'land_binary_mask'):
            o.set_config('environment:constant:%s' % v, 0)
        o.seed_elements(lon=4.0, lat=60.0, time=common.Fixture('rk4_3d_full').start, number=50, **{k: v.copy() for k, v in kw.items()})
    for k in ('orientation', 'length', 'height', 'draft', 'beam', 'wind_drag_coeff', 'water_drag_coeff', 'jibeProbability'):
        a, b = np.asarray(getattr(ours.elements_scheduled, k)), np.asarray(getattr(ref.elements_scheduled, k))
        assert a.dtype == b.dtype and np.array_equal(a, b), k
    assert ours.get_config('drift:max_speed') == 2 and ours.get_config('seed:orientation') == 'random'


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
    import shipdrift_host as sh
    import shipcases as cases
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    eng = sh.host_engine()
    E.default_engine = B.default_engine = lambda device=None: eng
    try:
        cases.run_product('wind_only', extra_config={'gpu:rng': 'philox'})
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
    assert all('ShipDrift' in r[2] for r in res)
