"""GPU: SedimentDrift (tests/sedimentcases.py: runs of the unmodified reference) on the device; the settling launch against the
per-iteration path with the Python bottom_interaction at 10^6 elements with both generators and at the block boundaries of the
launch; od_resuspend against the reference's expressions at the grid-stride boundaries of its launch; and a cell-sorted Philox run
against the unsorted one."""
import numpy as np
import pytest
import torch

import sedimentcases as sc
from test_sediment_host import _ref_resuspend, _resuspend_inputs, _same, run_scenario

pytestmark = pytest.mark.gpu


def _engine():
    from opendrift_b200.engine import default_engine
    return default_engine()


@pytest.mark.parametrize('case', list(sc.CASES))
def test_sediment_case_equals_the_reference(case):
    eng = _engine()
    before = eng.launches()
    o = sc.run_product(case)
    sc.check(o, case)
    assert eng.launches() > before


def _count_calls(eng, names):
    """Wraps the engine's mixing entry points to count them."""
    counts = {k: 0 for k in names}
    orig = {k: getattr(eng, k) for k in names}

    def wrap(k):
        def f(*a, **kw):
            counts[k] += 1
            return orig[k](*a, **kw)
        return f
    for k in names:
        setattr(eng, k, wrap(k))
    return counts, orig


@pytest.mark.parametrize('rng_kind', ['numpy', 'philox'])
@pytest.mark.parametrize('seed', [0, 1, 2, 6])
def test_settling_launch_equals_the_per_iteration_path_at_a_million(seed, rng_kind):
    eng = _engine()
    counts, orig = _count_calls(eng, ('vertical_mixing', 'vertical_mixing_settle'))
    try:
        a = run_scenario(seed, n=1_000_000, **{'gpu:rng': rng_kind})
        settle, redo = counts['vertical_mixing_settle'], counts['vertical_mixing']
        b = run_scenario(seed, per_iteration=True, n=1_000_000, **{'gpu:rng': rng_kind})
    finally:
        for k, f in orig.items():
            setattr(eng, k, f)
    assert settle == 5
    print(seed, rng_kind, 'per-iteration launches of the settling run', redo)
    _same(a, b)


@pytest.mark.parametrize('n', [1, 127, 128, 129, 255, 257, 4095, 4097])
def test_settling_launch_at_block_boundaries(n):
    """All elements released at once: the launch covers exactly n elements in blocks of 128 threads."""
    for seed in (0, 4):
        _same(run_scenario(seed, n=n, release=False), run_scenario(seed, per_iteration=True, n=n, release=False))


def test_resuspend_at_the_grid_stride_boundaries():
    """The launch is capped at 8 blocks of 256 threads per SM; every thread then loops over the elements."""
    eng = _engine()
    span = eng.lib.od_device_sm_count(eng.ctx) * 8 * 256
    for k, n in enumerate((1, 255, 256, 257, span - 1, span, span + 1, 2 * span + 17, 10_000_000)):
        thr = (0.2, 0.5, 0.0)[k % 3]
        u, v, moving, z = _resuspend_inputs(k, n, thr)
        for zt in (np.float32, np.float64):
            zz = z.astype(zt)
            want_m, want_z = _ref_resuspend(u, v, thr, moving, zz)
            dm, dz = eng.to_device(moving.copy()), eng.to_device(zz.copy())
            eng.resuspend(eng.to_device(u), eng.to_device(v), thr, dm, dz)
            assert np.array_equal(dm.cpu().numpy(), want_m)
            gz = dz.cpu().numpy()
            assert np.array_equal(gz, want_z, equal_nan=True) and np.array_equal(np.signbit(gz), np.signbit(want_z))


def test_cell_sorted_run_equals_the_unsorted_one():
    """10^6 elements with the device generator, re-ordered by cell every step: the result per element ID equals that of the run
    without the sort (the draws are keyed by element ID, the settling decisions are per element)."""
    eng = _engine()
    sorts = []
    plain_sort = eng.sort_by_cell

    def counting_sort(*a, **k):
        sorts.append(1)
        return plain_sort(*a, **k)
    eng.sort_by_cell = counting_sort
    try:
        o0 = run_scenario(6, n=1_000_000, **{'gpu:rng': 'philox', 'gpu:sort_interval_steps': 0})
        assert not sorts
        o1 = run_scenario(6, n=1_000_000, **{'gpu:rng': 'philox', 'gpu:sort_interval_steps': 1})
        assert len(sorts) >= 3
    finally:
        del eng.sort_by_cell
    e0, e1 = o0.elements, o1.elements
    a, b = np.argsort(np.asarray(e0.ID)), np.argsort(np.asarray(e1.ID))
    for k in ('ID', 'lon', 'lat', 'z', 'moving', 'status'):
        assert np.array_equal(np.asarray(getattr(e0, k))[a], np.asarray(getattr(e1, k))[b], equal_nan=True), k
    assert (np.asarray(e0.moving) == 0).sum() > 0
