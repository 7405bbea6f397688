"""GPU: LarvalFish (tests/larvalcases.py: runs of the unmodified reference) on the device, with the launches each
step makes; the two launches against their host build at 10^6 elements and at the grid-stride boundaries; and a cell-sorted Philox
run against the unsorted one."""
import numpy as np
import pytest
import torch

import larvalcases as lc
import larval_host
from test_larval_host import _random_elements, _random_environment, _edge_cases, _launch

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


@pytest.mark.parametrize('case', list(lc.CASES) + [lc.EXAMPLE])
def test_larval_case_equals_the_reference(case):
    eng = _engine()
    calls, restore = _counting(eng, ('larval_develop', 'larval_migrate', 'vertical_mixing'))
    try:
        o, err = lc.run_product(case)
    finally:
        restore()
    worst = lc.check(o, case, err)
    print(case, worst)
    if case in lc.RAISES:
        assert isinstance(err, ValueError) and calls['larval_develop'] == 1
        return
    steps = len(np.load(lc.GOLDEN)['%s__h_len' % case])
    mixing = case == lc.EXAMPLE or lc.CASES[case][0].get('drift:vertical_mixing', True)
    assert calls['larval_develop'] == steps * (2 if case == 'subclass_reference_update' else 1)
    assert calls['larval_migrate'] == steps
    assert calls['vertical_mixing'] == (steps if mixing else 0)          # one fused launch per step, no per-iteration mixing


def _same(eng, n, seed, f64):
    rng = np.random.default_rng(seed)
    el = _random_elements(n, rng, set(f64))
    t, s = _random_environment(n, rng)
    _edge_cases(el, t, s, 3600.0)
    got, flags = _launch(eng, el, t, s, 3600.0, 13, 0.3, dev=eng.device)
    host, hflags = _launch(larval_host.host_engine(), el, t, s, 3600.0, 13, 0.3)
    assert flags == hflags
    assert np.array_equal(got['hatched'], host['hatched'])
    # Both sides run the same code: float64 functions (CUDA's, glibc's) rounded where NumPy works in float32, no contraction.  The
    # float64 functions may differ by an ulp; that reaches a float32 result only when the value lies next to a float32 rounding
    # boundary, so float32 outputs are equal but for a rare element one ulp apart, and float64 outputs stay well within one
    # float32 ulp.
    stats = {}
    for k in ('stage_fraction', 'weight', 'length', 'terminal_velocity', 'z'):
        a, b = got[k], host[k]
        assert a.dtype == b.dtype, k
        f = np.isfinite(b)
        assert np.array_equal(np.isfinite(a), f) and np.array_equal(a[~f], b[~f], equal_nan=True), k
        ulps = np.abs(a[f].astype(np.float64) - b[f]) / np.spacing(np.abs(b[f]).astype(np.float32)).astype(np.float64)
        differing = int(np.count_nonzero(a[f] != b[f]))
        stats[k] = (str(a.dtype), float(ulps.max(initial=0.0)), differing)
        assert ulps.max(initial=0.0) <= 1.0, (k, stats[k])
        if a.dtype == np.float32:
            assert differing <= max(2, n // 10000), (k, stats[k])
    print(n, f64, stats)


@pytest.mark.parametrize('f64', [(), ('weight', 'length', 'diameter', 'neutral_buoyancy_salinity', 'z', 'hatched', 'stage_fraction')])
def test_launches_equal_their_host_build_at_1e6_elements(f64):
    _same(_engine(), 1_000_000, 21, f64)


def test_launches_equal_their_host_build_at_the_grid_stride_boundaries():
    eng = _engine()
    sm = torch.cuda.get_device_properties(eng.device).multi_processor_count
    block = 128                                 # OD_BLOCK (csrc/od_ctx.cuh)
    full = sm * 8 * block                       # one pass of the capped grid
    for n in (1, block - 1, block, block + 1, full - 1, full, full + 1, 2 * full + 3):
        _same(eng, n, n, ('length', 'z'))


def test_cell_sorted_philox_run_equals_the_unsorted_one():
    kw = {'gpu:rng': 'philox'}
    runs = []
    for interval in (0, 1):
        o, err = lc.run_product('ts_arrays_hatching', extra_config=dict(kw, **{'gpu:sort_interval_steps': interval}), n=200_000)
        assert err is None
        runs.append(lc.summary(o))
    a, b = runs
    ia, ib = np.argsort(a['id']), np.argsort(b['id'])
    assert np.array_equal(a['id'][ia], b['id'][ib])
    for k in ('lon', 'lat') + lc.VARS:
        assert np.array_equal(a[k][ia], b[k][ib], equal_nan=True), k
