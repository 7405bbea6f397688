"""GPU: gridded readers on a rotated-pole grid (tests/rotpolecases.py: runs of the unmodified reference) through the drop-in models --
the rotation of positions, the coverage and index rules of rotated longitudes, and the rotation of vector components, on the
device; and a cell-sorted run on a rotated grid against the unsorted one."""
import numpy as np
import pytest

import rotpolecases as rc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('case', list(rc.CASES))
def test_rotated_pole_case_equals_the_reference(case):
    o = rc.run_product(case)
    e, dz, moved = rc.check(o, case)
    assert moved > 5e-3
    assert e < 5e-8 and dz <= (1e-9 if 'mixing' in case else 1e-5), (e, dz)
    ref = np.load(rc.GOLDEN)
    lon0, lat0 = rc.setup(case)[6:8]
    assert rc.unmoved(o.elements.lon, o.elements.lat, lon0, lat0) == int(ref['%s__unmoved' % case])


def test_cell_sort_on_a_rotated_grid_changes_nothing(monkeypatch):
    from opendrift_b200.engine import default_engine
    eng = default_engine()
    sorts = []
    plain = eng.sort_by_cell

    def counting(*a, **k):
        sorts.append(1)
        return plain(*a, **k)
    monkeypatch.setattr(eng, 'sort_by_cell', counting)
    o0 = rc.run_many(0)
    assert not sorts
    o1 = rc.run_many(1)
    assert len(sorts) >= 3
    e0, e1 = o0.elements, o1.elements
    assert len(e0.ID) == len(e1.ID) >= 100000
    a, b = np.argsort(np.asarray(e0.ID)), np.argsort(np.asarray(e1.ID))
    for k in ('ID', 'lon', 'lat', 'z', 'status'):
        assert np.array_equal(np.asarray(getattr(e0, k))[a], np.asarray(getattr(e1, k))[b], equal_nan=True), k
