"""GPU: drift:use_tabularised_stokes_drift (tests/stokestabcases.py: runs of the unmodified reference) through the drop-in
OceanDrift on the device; od_stokes_parameterised bit for bit against the reference's expressions at benchmark scale and at the
grid-stride boundaries of its launch; and a cell-sorted run of 10^6 elements against the unsorted one."""
import numpy as np
import pytest
import torch

import common
import stokestabcases as sc
from test_stokestab_host import _ref_parameterised, _winds
from opendrift_b200.models.environment import stokes_coefficients

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('case', list(sc.CASES))
def test_tabularised_stokes_case_equals_the_reference(case):
    o = sc.run_product(case)
    print(case, sc.check(o, case))


def _check_kernel(eng, n, fetch, seed):
    xw, yw = _winds(seed, n)
    want = _ref_parameterised(xw, yw, fetch)
    cw, ch = stokes_coefficients(fetch)
    dx, dy = eng.to_device(xw), eng.to_device(yw)
    us, vs, hs = (torch.full((n,), 7.0, dtype=torch.float32, device=eng.device) for _ in range(3))
    eng.stokes_parameterised(dx, dy, cw, ch, us, vs, hs)
    for got, w in zip((us, vs, hs), want):
        g = got.cpu().numpy()
        assert np.array_equal(g, w, equal_nan=True)
        assert np.array_equal(np.signbit(g), np.signbit(w))


def test_parameterisation_equals_numpy_at_ten_million_elements():
    from opendrift_b200.engine import default_engine
    eng = default_engine()
    for fetch in ('5000', '25000', '50000'):
        _check_kernel(eng, 10_000_000, fetch, 3)


def test_parameterisation_at_the_grid_stride_boundaries():
    """The launch is capped at 8 blocks of 256 threads per SM; every thread then loops over the elements."""
    from opendrift_b200.engine import default_engine
    eng = default_engine()
    span = eng.lib.od_device_sm_count(eng.ctx) * 8 * 256
    for k, n in enumerate((1, 16, 255, 256, 257, span - 1, span, span + 1, 2 * span - 1, 2 * span + 17, 3 * span)):
        _check_kernel(eng, n, ('5000', '25000', '50000')[k % 3], k)


def test_cell_sorted_run_equals_the_unsorted_one():
    """10^6 elements with the device generator: the arrays are re-ordered by cell every step, after the parameterisation has
    taken its maxima over all elements; the result per element ID equals that of the run without the sort."""
    from opendrift_b200.engine import default_engine
    from opendrift_b200.models.oceandrift import OceanDrift
    from opendrift_b200.readers import reader_regular_grid
    eng = default_engine()
    sorts = []
    plain_sort = eng.sort_by_cell

    def counting_sort(*a, **k):
        sorts.append(1)
        return plain_sort(*a, **k)

    def run(sort_every):
        fx = common.Fixture('rk4_3d_full')
        mk = lambda f, name, z=None, lon=fx.grid_lon, lat=fx.grid_lat: reader_regular_grid.Reader(lon, lat, z, fx.times, f,  # noqa: E731
                                                                                                  name=name)
        o = OceanDrift(loglevel=50)
        o.add_reader(mk({common.CUR[0]: fx.u, common.CUR[1]: fx.v, 'upward_sea_water_velocity': (20 * fx.w).astype(np.float32)},
                        'current', fx.grid_z))
        o.add_reader(mk({'x_wind': fx.x_wind, 'y_wind': fx.y_wind}, 'wind', lon=fx.wind_lon, lat=fx.wind_lat))
        for k, v in {'general:use_auto_landmask': False, 'environment:constant:land_binary_mask': 0, 'seed:ocean_only': False,
                     'drift:use_tabularised_stokes_drift': True, 'drift:advection_scheme': 'runge-kutta4', 'gpu:rng': 'philox',
                     'gpu:sort_interval_steps': sort_every}.items():
            o.set_config(k, v)
        rng = np.random.default_rng(5)
        n = 1_000_000
        o.seed_elements(lon=rng.uniform(2.3, 3.7, n), lat=rng.uniform(56.2, 56.9, n), z=-rng.uniform(0, 20, n).astype(np.float32),
                        time=fx.start)
        o.run(steps=4, time_step=sc.DT, time_step_output=sc.DT)
        return o

    eng.sort_by_cell = counting_sort
    try:
        o0 = run(0)
        assert not sorts
        o1 = run(1)
        assert len(sorts) >= 3
    finally:
        del eng.sort_by_cell
    e0, e1 = o0.elements, o1.elements
    a, b = np.argsort(np.asarray(e0.ID)), np.argsort(np.asarray(e1.ID))
    for k in ('ID', 'lon', 'lat', 'z'):
        assert np.array_equal(np.asarray(getattr(e0, k))[a], np.asarray(getattr(e1, k))[b], equal_nan=True), k
    assert len(a) == 1_000_000
