"""GPU: the work at a reader-time change and the cell sort.

- Pair texels built ahead on the copy stream (FieldGroup.prefetch -> od_group_prepare_pair) give the same positions, bit for
  bit, as pair texels built on demand in front of the first step that needs them (prefetch off), forward and backward, across
  several reader hours.
- od_sort_by_cell (warp-aggregated bin counts and scatter) returns a permutation along which the (level, 4x4-cell tile) key
  never decreases, for 10 M elements, for a partially covered grid (key 0 first) and for fewer elements than one warp."""
from datetime import timedelta

import numpy as np
import pytest

from opendrift_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


def _run(prefetch, backward, steps=40, n=200_000):
    import torch
    from opendrift_b200.engine import Engine
    eng = Engine(0)
    grid = syn.GridSpec(nx=96, ny=80, nz=6)
    times = syn.slab_times(12)
    slabs = [tuple(torch.from_numpy(a).cuda() for a in syn.double_gyre_uv(grid, (t - syn.T0).total_seconds())) for t in times]
    w = torch.from_numpy(syn.upward_w(grid)).cuda()
    grp = eng.add_group(grid.lon, grid.lat, grid.z, 2, times, lambda ti, c: slabs[ti][c], (0.0, 0.0), n_slots=3)
    wgrp = eng.add_group(grid.lon, grid.lat, grid.z, 1, times, lambda ti, c: w, (0.0,), n_slots=3)
    grp.prefetch_on = wgrp.prefetch_on = prefetch
    rng = np.random.default_rng(7)
    lon = torch.from_numpy(rng.uniform(grid.lon[8], grid.lon[-8], n)).cuda()
    lat = torch.from_numpy(rng.uniform(grid.lat[8], grid.lat[-8], n)).cuda()
    z = torch.from_numpy(rng.uniform(-9.0, -0.5, n).astype(np.float32)).cuda()
    dt = timedelta(seconds=-600 if backward else 600)
    eng.direction = -1 if backward else 1
    t = times[-1] if backward else times[0]
    for k in range(steps):
        if k % 7 == 0:                     # the cell sort between steps, as run() and the benchmark do
            perm = eng.sort_by_cell(grp, lon, lat, z)
            lon, lat, z = (eng.permute(perm, a) for a in (lon, lat, z))
        eng.step_oceandrift(grp, 'runge-kutta4', t, dt, lon, lat, z, w_group=wgrp, pos_f32=(k == 0))
        t += dt
    torch.cuda.synchronize()
    out = [a.cpu().numpy() for a in (lon, lat, z)]
    eng.close()
    # element order after the sorts may differ between runs: compare as sets of records
    rec = np.stack([out[0], out[1], out[2].astype(np.float64)], axis=1)
    return rec[np.lexsort(rec.T[::-1])]


@pytest.mark.parametrize('backward', [False, True])
def test_pairs_built_ahead_equal_pairs_built_on_demand(backward):
    ahead = _run(True, backward)
    on_demand = _run(False, backward)
    assert np.array_equal(ahead, on_demand)
    assert np.isfinite(ahead).all()


def _keys(grid, lon, lat):
    """The sort key of a 2-D group for positions well inside cells: 1 + tile row * tiles per row + tile column, 0 outside."""
    dx = float(grid.lon[1]) - float(grid.lon[0])
    dy = float(grid.lat[1]) - float(grid.lat[0])
    ix = np.floor((lon - float(grid.lon[0])) / dx).astype(np.int64)
    iy = np.floor((lat - float(grid.lat[0])) / dy).astype(np.int64)
    inside = (ix >= 0) & (ix < grid.nx - 1) & (iy >= 0) & (iy < grid.ny - 1)
    ntx = (grid.nx + 3) // 4
    return np.where(inside, 1 + (iy // 4) * ntx + ix // 4, 0)


@pytest.mark.parametrize('n,outside', [(10_000_000, 0.0), (1_000_000, 0.3), (1, 0.0), (5, 0.4), (31, 0.5), (33, 0.0)])
def test_cell_sort_is_a_permutation_with_non_decreasing_keys(n, outside):
    import torch
    from opendrift_b200.engine import Engine
    eng = Engine(0)
    grid = syn.GridSpec(nx=300, ny=200, nz=1)
    grp = eng.add_group(grid.lon, grid.lat, None, 2, syn.slab_times(2), lambda ti, c: None, (0.0, 0.0), n_slots=2)
    rng = np.random.default_rng(n)
    # cell centres with a jitter of a quarter cell: the cell of every element is unambiguous
    ix = rng.integers(0, grid.nx - 1, n)
    iy = rng.integers(0, grid.ny - 1, n)
    lon = float(grid.lon[0]) + (ix + 0.5 + rng.uniform(-0.25, 0.25, n)) * (float(grid.lon[1]) - float(grid.lon[0]))
    lat = float(grid.lat[0]) + (iy + 0.5 + rng.uniform(-0.25, 0.25, n)) * (float(grid.lat[1]) - float(grid.lat[0]))
    away = rng.random(n) < outside
    lon[away] -= 10.0                                # outside the grid: key 0
    if n >= 1_000_000:                               # arrive roughly cell-sorted, as the benchmark's elements do
        o = np.argsort(_keys(grid, lon, lat) * 4 + rng.integers(0, 4, n), kind='stable')
        lon, lat = lon[o], lat[o]
    perm = eng.sort_by_cell(grp, torch.from_numpy(lon).cuda(), torch.from_numpy(lat).cuda()).cpu().numpy()
    eng.close()
    assert perm.shape == (n,)
    assert np.array_equal(np.sort(perm), np.arange(n))
    k = _keys(grid, lon, lat)[perm]
    assert (np.diff(k) >= 0).all()
    assert (k == 0).sum() == away.sum()

