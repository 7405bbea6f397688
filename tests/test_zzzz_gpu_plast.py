"""GPU: PlastDrift (tests/plastcases.py: runs of the unmodified reference) on the device, with the launches each step makes; the launch
against its host build at 10^6 elements and at the grid-stride boundaries of the launch; and a cell-sorted Philox run against the
unsorted one."""
import numpy as np
import pytest
import torch

import common
import plastcases as pc
import plast_host
from test_plast_host import _random_inputs, _special_scales

pytestmark = pytest.mark.gpu


def _engine():
    from opendrift_b200.engine import default_engine
    return default_engine()


def _counting(eng, names):
    calls = {k: 0 for k in names}
    orig = {k: getattr(eng, k) for k in names}

    def wrap(k):
        def f(*a, **kw):
            calls[k] += 1
            return orig[k](*a, **kw)
        return f
    for k in names:
        setattr(eng, k, wrap(k))
    return calls, lambda: [setattr(eng, k, v) for k, v in orig.items()]


@pytest.mark.parametrize('case', list(pc.CASES))
def test_plast_case_equals_the_reference(case):
    eng = _engine()
    calls, restore = _counting(eng, ('plast_step', 'vertical_mixing', 'stokes_drift'))
    try:
        o = pc.run_product(case)
    finally:
        restore()
    err, zerr = pc.check(o, case)
    print('%s: max position difference %.2e deg, depth %.2e m' % (case, err, zerr))
    assert calls['plast_step'] == pc.STEPS
    assert calls['vertical_mixing'] == (pc.STEPS if case in pc.RANDOMWALK else 0)
    if case != 'subclass_reference_update':
        assert calls['stokes_drift'] == 0


def test_wind_drift_shear_known_answer():
    from opendrift_b200.models.plastdrift import PlastDrift
    _engine()
    lon, lat = pc.run_shear(PlastDrift)
    np.testing.assert_array_almost_equal(lon, pc.SHEAR_LON)
    ref = np.load(pc.GOLDEN)
    assert max(common.max_err_deg(lon, lat, ref['shear__lon'], ref['shear__lat'])) < pc.TOL_DEG


def _launch(eng, n, seed, profile='Phillips', wdd=0.1, dtypes=(False, True, False)):
    """One launch on the device and one on the host build from the same inputs and draws: (lon, lat, z) of each"""
    rng = np.random.default_rng(seed)
    el, env = _random_inputs(n, rng, *dtypes)
    _special_scales(el, env)
    lon0, lat0 = rng.uniform(-10, 10, n), rng.uniform(50, 70, n)
    draws = rng.standard_exponential(n)
    out = []
    for e, dev in ((eng, eng.device), (plast_host.host_engine(), torch.device('cpu'))):
        t = {k: torch.from_numpy(v.copy()).to(dev) for k, v in env.items()}
        lon, lat = torch.tensor(lon0, device=dev), torch.tensor(lat0, device=dev)
        sub = (t['ocean_vertical_diffusivity'], torch.from_numpy(el['terminal_velocity'].copy()).to(dev),
               torch.from_numpy(draws).to(dev), torch.arange(n, dtype=torch.int32, device=dev), 0, 0)
        z = e.plast_step(lon, lat, torch.from_numpy(el['moving'].copy()).to(dev), torch.from_numpy(el['z'].copy()).to(dev), 3600.0,
                         submerge=sub, stokes=(t['sea_surface_wave_stokes_drift_x_velocity'], t['sea_surface_wave_stokes_drift_y_velocity'],
                                               t['sea_surface_wave_significant_height'], t['x_wind'], t['y_wind'], 0, profile, None),
                         wind=(t['x_wind'], t['y_wind'], torch.from_numpy(el['wind_drift_factor'].copy()).to(dev), wdd))
        out.append((lon.cpu().numpy(), lat.cpu().numpy(), z.cpu().numpy()))
    return out


def _same(out):
    (dl, da, dz), (hl, ha, hz) = out
    # the depths: one float32 (or float64) division and one float64 product, bit for bit
    assert np.array_equal(dz, hz, equal_nan=True)
    # CUDA's exp / erfc / atan2 / atan2f against glibc's differ by an ulp here and there (a float32 ulp of the wind move's azimuth, with
    # wind_drift_depth = 0 and a float32 wind_drift_factor, is a few 1e-4 m after an hour): the moves agree within 2 mm
    f = np.isfinite(dz)
    lat0 = np.radians(ha[f])
    err_m = np.hypot((dl[f] - hl[f]) * np.cos(lat0) * 111320.0, (da[f] - ha[f]) * 110574.0)
    assert err_m.max() < 2e-3, err_m.max()
    assert np.array_equal(np.isnan(dl), np.isnan(hl))


@pytest.mark.parametrize('wdd', [0.1, 0.0])
def test_launch_equals_its_host_build_at_1e6_elements(wdd):
    _same(_launch(_engine(), 1_000_000, 21, wdd=wdd))


def test_launch_equals_its_host_build_at_the_grid_stride_boundaries():
    eng = _engine()
    sm = torch.cuda.get_device_properties(eng.device).multi_processor_count
    block = 128                                 # OD_BLOCK (csrc/od_ctx.cuh)
    full = sm * 8 * block                       # one pass of the capped grid
    for n in (1, block - 1, block, block + 1, full - 1, full, full + 1, 2 * full + 3):
        _same(_launch(eng, n, n, profile='exponential', dtypes=(True, False, True)))


def test_cell_sorted_philox_run_equals_the_unsorted_one():
    kw = {'gpu:rng': 'philox'}
    runs = []
    for interval in (0, 1):
        o = pc.run_product('k_profile', extra_config=dict(kw, **{'gpu:sort_interval_steps': interval}), n=200_000)
        runs.append(pc.summary(o))
    a, b = runs
    ia, ib = np.argsort(a['id']), np.argsort(b['id'])
    assert np.array_equal(a['id'][ia], b['id'][ib])
    assert np.array_equal(a['z'][ia], b['z'][ib])
    assert np.array_equal(a['lon'][ia], b['lon'][ib]) and np.array_equal(a['lat'][ia], b['lat'][ib])
