"""GPU: the specialised step kernel (csrc/od_spec.cuh) against the general step kernel (OD_OPT_SPEC off), BIT FOR BIT on lon, lat
and z, on forcing fields whose texels are not all ordinary numbers: land values the NaN fill leaves, +-inf texels, +-0,
subnormal and near-FLT_MAX texels, and reader times that go from pairs without NaNs to pairs with NaNs and back (the pair cache
re-packs its entries on the way).  Also the benchmarked configuration, sorted and unsorted."""
from datetime import timedelta

import numpy as np
import pytest

import bigcases as bc
from opendrift_b200 import synthetic as syn
from test_zz_gpu_spec import _run, _same

pytestmark = pytest.mark.gpu

FLT_MAX = np.float32(3.4028235e38)


@pytest.mark.parametrize('sort', [0, 20])
def test_spec_equals_general_kernel_on_the_benchmarked_configuration(sort):
    if 'cfg2' not in bc.KINDS:
        pytest.skip('fixture not generated')
    c = bc.BigCase('cfg2')

    def make():
        o = c.model(**{'gpu:sort_interval_steps': sort})
        o._test_run_args = dict(steps=c.steps, time_step=c.dt, time_step_output=c.steps * c.dt)
        return o

    _same(_run(make, True), _run(make, False))


GRID = dict(nx=96, ny=80, nz=6, lon0=0.0, dlon=0.05, lat0=55.0, dlat=0.025, dz=4.0)


def _fields(kind, nt, seed):
    """u, v, w slabs (nt, nz, ny, nx) float32 for one case, and whether the NaN fill runs on upload."""
    g = syn.GridSpec(**GRID)
    times = [syn.T0 + timedelta(hours=h) for h in range(nt)]
    uv = [syn.double_gyre_uv(g, (t - syn.T0).total_seconds()) for t in times]
    u = np.stack([a for a, _ in uv])
    v = np.stack([b for _, b in uv])
    w = np.stack([syn.upward_w(g)] * nt)
    rng = np.random.default_rng(seed)
    fill = True
    if kind == 'land':                          # a block wider than 2 x 10 fill passes: its middle stays NaN
        for a in (u, v, w):
            a[:, :, 20:60, 30:70] = np.nan
    elif kind == 'inf':                         # no fill: the infinities reach the pair texels
        fill = False
        for a in (u, v, w):
            m = rng.random(a.shape) < 0.002
            a[m] = np.where(rng.random(m.sum()) < 0.5, np.inf, -np.inf)
    elif kind == 'extreme':                     # finite, but at the ends of the float32 range
        special = np.array([0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -1.1754942e-38, 1.17549435e-38, FLT_MAX, -FLT_MAX,
                            np.float32(3.4028233e38), np.float32(-1e37)], np.float32)
        for a, p in ((u, 0.003), (v, 0.003), (w, 0.02)):
            m = rng.random(a.shape) < p
            a[m] = rng.choice(special, m.sum())
        tiny = rng.random(u.shape) < 0.05       # subnormal and zero velocities over whole patches
        u[tiny] = np.float32(1e-41)
        v[tiny] = -0.0
    elif kind == 'switch':                      # reader time 2 has land that survives the fill, the others none
        for a in (u, v):
            a[2, :, 20:60, 30:70] = np.nan
    return g, times, u, v, w, fill


def _engine_run(kind, nt, steps, seed=3, n=60_000):
    """The same particles stepped with the specialised kernel and with the general one (fused RK4 + vertical advection)."""
    from opendrift_b200.engine import default_engine
    eng = default_engine()
    g, times, u, v, w, fill = _fields(kind, nt, seed)
    rng = np.random.default_rng(seed + 1)
    lon0 = rng.uniform(float(g.lon[0]) - 0.1, float(g.lon[-1]) + 0.1, n)
    lat0 = rng.uniform(float(g.lat[0]) - 0.05, float(g.lat[-1]) + 0.05, n)
    z0 = rng.uniform(-22.0, 0.0, n).astype(np.float32)
    z0[::5] = 0.0
    grp = eng.add_group(g.lon, g.lat, g.z, 2, times, lambda ti, c: (u, v)[c][ti], (0.3, -0.2))
    wgrp = eng.add_group(g.lon, g.lat, g.z, 1, times, lambda ti, c: w[ti], (0.0,))
    if not fill:
        grp.fill_nan = wgrp.fill_nan = 0
    out = []
    try:
        for on in (True, False):
            eng.set_spec(on)
            lon, lat, z = eng.to_device(lon0), eng.to_device(lat0), eng.to_device(z0)
            t, dt = times[0], timedelta(seconds=600)
            for _ in range(steps):
                eng.step_oceandrift(grp, 'runge-kutta4', t, dt, lon, lat, z, w_group=wgrp)
                t += dt
            eng.sync()
            out.append((lon.cpu().numpy(), lat.cpu().numpy(), z.cpu().numpy()))
    finally:
        eng.set_spec(True)
        eng.free_group(grp)
        eng.free_group(wgrp)
    return out


def _bitwise(a, b):
    for x, y in zip(a, b):
        assert x.dtype == y.dtype
        assert np.array_equal(np.isnan(x), np.isnan(y))
        f = ~np.isnan(x)
        assert np.array_equal(x[f].view(np.uint8), y[f].view(np.uint8))


@pytest.mark.parametrize('kind', ['finite', 'land', 'inf', 'extreme'])
def test_spec_equals_general_kernel_on_unusual_texels(kind):
    spec, gen = _engine_run(kind, nt=3, steps=10)
    _bitwise(spec, gen)
    assert np.isfinite(spec[0]).mean() > 0.5            # most particles still have a position to compare


def test_pairs_turning_non_finite_and_back():
    # 7 reader times, 36 steps: 6 distinct pairs through a cache of 4 entries, so entries that held a pair with NaNs are
    # re-packed with pairs without them and the other way round
    spec, gen = _engine_run('switch', nt=7, steps=36)
    _bitwise(spec, gen)
