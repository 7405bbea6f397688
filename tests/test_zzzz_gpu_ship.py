"""GPU: ShipDrift (tests/shipcases.py: runs of the unmodified reference) on the device; the launch against its host build at 10^6
ships and at the grid-stride boundaries of the launch; one launch per step; and a cell-sorted Philox run against the unsorted one."""
import numpy as np
import pytest
import torch

import common
import shipcases as sc
import shipdrift_host
from test_ship_host import _random_inputs, _table

pytestmark = pytest.mark.gpu


def _engine():
    from opendrift_b200.engine import default_engine
    return default_engine()


def _counting(eng):
    calls = []
    orig = eng.ship_step

    def f(*a, **kw):
        calls.append(1)
        return orig(*a, **kw)
    eng.ship_step = f
    return calls, lambda: setattr(eng, 'ship_step', orig)


@pytest.mark.parametrize('case', list(sc.CASES))
def test_ship_case_equals_the_reference(case):
    eng = _engine()
    calls, restore = _counting(eng)
    try:
        o = sc.run_product(case)
    finally:
        restore()
    err = sc.check(o, case)
    print('%s: max position difference %.2e deg' % (case, err))
    assert len(calls) == (0 if case == 'subclass_reference_update' else sc.STEPS)


def _launch(eng, n, period, stokes, seed):
    """One launch on the device and one on the host build from the same inputs: (device lon, lat, status), (host ...)"""
    rng = np.random.default_rng(seed)
    el, env = _random_inputs(n, rng, period)
    wf, ipF, ipD, table = _table()
    lon0, lat0 = rng.uniform(-10, 10, n), rng.uniform(50, 70, n)
    T = env[sc.TM02]
    tm_wind = not T.max() > 0
    fill = np.mean(T[T > 0]) if not tm_wind and T.min() == 0 else None
    hs_wind = not env['sea_surface_wave_significant_height'].max() > 0
    out = []
    for e, dev in ((eng, eng.device), (shipdrift_host.host_engine(), torch.device('cpu'))):
        t = {k: torch.from_numpy(v.copy()).to(dev) for k, v in env.items()}
        envd = {'x_sea_water_velocity': t[common.CUR[0]], 'y_sea_water_velocity': t[common.CUR[1]], 'x_wind': t['x_wind'],
                'y_wind': t['y_wind'], 'hs': t['sea_surface_wave_significant_height'], 'period': t[sc.TM02],
                'stokes_x': t['sea_surface_wave_stokes_drift_x_velocity'] if stokes else None,
                'stokes_y': t['sea_surface_wave_stokes_drift_y_velocity'] if stokes else None, 'land_binary_mask': t['land_binary_mask']}
        lon, lat = torch.tensor(lon0, device=dev), torch.tensor(lat0, device=dev)
        status = torch.zeros(n, dtype=torch.int32, device=dev)
        moving = torch.ones(n, dtype=torch.int32, device=dev)
        eld = {k: torch.from_numpy(el[k].copy()).to(dev) for k in ('length', 'height', 'draft', 'beam', 'wind_drag_coeff', 'water_drag_coeff')}
        tab = tuple(torch.from_numpy(a).to(dev) for a in table[:2]) + (table[2],)
        st = e.ship_step(lon, lat, moving, status, eld, torch.from_numpy(el['orientation'].copy()).to(dev), envd, tab, 3600.0,
                         hs_wind=hs_wind, tm_wind=tm_wind, tm_fill=fill, strand_code=3)
        out.append((lon.cpu().numpy(), lat.cpu().numpy(), status.cpu().numpy(), moving.cpu().numpy(), envd['hs'].cpu().numpy(),
                    envd['period'].cpu().numpy(), st))
    return out, lon0, lat0


def _same(out, lon0, lat0):
    (dl, da, ds, dm, dh, dp, dst), (hl, ha, hs, hm, hh, hp, hst) = out
    assert np.array_equal(ds, hs) and np.array_equal(dm, hm) and dst == hst
    # Hs from the wind is float32 arithmetic, bit for bit; the period from the wind is a float64 division, bit for bit
    assert np.array_equal(dh, hh) and np.array_equal(dp, hp)
    # CUDA's float64 exp / pow / cos / atan2 against glibc's differ by an ulp here and there; rounded to float32 in the spectrum, that
    # can be one float32 ulp of a spectrum value: the moves of an hour differ by up to 0.7 mm at 10^6 ships on an H100
    err_m = np.hypot((dl - hl) * np.cos(np.radians(lat0)) * 111320.0, (da - ha) * 110574.0)
    assert err_m.max() < 2e-3, err_m.max()


@pytest.mark.parametrize('period', ['wind', 'reader', 'partial'])
def test_launch_equals_its_host_build_at_1e6_ships(period):
    _same(*_launch(_engine(), 1_000_000, period, period == 'reader', 21))


def test_launch_equals_its_host_build_at_the_grid_stride_boundaries():
    eng = _engine()
    sm = torch.cuda.get_device_properties(eng.device).multi_processor_count
    full = sm * 8 * 256                     # one pass of the capped grid
    for n in (1, 255, 256, 257, full - 1, full, full + 1, 2 * full + 3):
        _same(*_launch(eng, n, 'reader', True, n))


def test_cell_sorted_philox_run_equals_the_unsorted_one():
    kw = {'gpu:rng': 'philox', 'environment:fallback:horizontal_diffusivity': 100}
    runs = []
    for interval in (0, 1):
        o = sc.run_product('waves_hs_tm02', extra_config=dict(kw, **{'gpu:sort_interval_steps': interval}), n=200_000)
        runs.append(sc.summary(o))
    a, b = runs
    ia, ib = np.argsort(a['id']), np.argsort(b['id'])
    assert np.array_equal(a['id'][ia], b['id'][ib])
    assert np.array_equal(a['lon'][ia], b['lon'][ib]) and np.array_equal(a['lat'][ia], b['lat'][ib])
