"""A varying sea surface height (tests/sealevelcases.py) on the host build of the device sources: the drop-in OceanDrift with sea
floor, sea surface height and diffusivity readers against runs of the unmodified reference; and the per-element functions of
csrc/od_sealevel.cuh against the reference's NumPy expressions restated here."""
import numpy as np
import pytest
import torch

import sealevelcases as sc
import sealevel_host


@pytest.fixture()
def host_engine(monkeypatch):
    eng = sealevel_host.host_engine()
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    monkeypatch.setattr(E, 'default_engine', lambda device=None: eng)
    monkeypatch.setattr(B, 'default_engine', lambda device=None: eng)
    yield eng


@pytest.mark.parametrize('case', list(sc.CASES))
def test_sea_level_case_equals_the_reference(case, host_engine):
    o = sc.run_product(case)
    sc.check(o, case)
    calls = host_engine.lib.calls
    if case.startswith('correction'):
        assert 'od_vertical_advection_corrected' in calls and 'od_store_previous_env' in calls
    if case.startswith('mixing'):
        assert 'od_vertical_mixing' in calls
    if case == 'correction_release_east':
        ref = np.load(sc.GOLDEN)
        cats = [str(c) for c in ref[case + '__cats']]
        assert 'missing_data' in cats and (ref[case + '__d_status'] == cats.index('missing_data')).sum() > 0
    if case == 'mixing_bottom_hook':
        assert len(o.zmins) > 0


def test_sea_surface_height_reader_alone_changes_nothing(host_engine):
    """A sea_surface_height reader with the default configuration (no sea-floor reader, no mixing, no correction): the same
    result, bit for bit, as the run without it, and still the fused step."""
    from opendrift_b200.models.oceandrift import OceanDrift
    from opendrift_b200.readers import reader_regular_grid
    mk = lambda lon, lat, z, t, f, name: reader_regular_grid.Reader(lon, lat, z, t, f, name=name)      # noqa: E731
    o1 = sc.run_case('default_ssh_only', OceanDrift, mk)
    n_fused = host_engine.lib.calls.count('od_step_oceandrift')
    assert n_fused == sc.STEPS
    host_engine.lib.calls.clear()
    saved = sc.CASES['default_ssh_only']
    try:
        sc.CASES['default_ssh_only'] = (saved[0], (), saved[2], saved[3], saved[4])
        o2 = sc.run_case('default_ssh_only', OceanDrift, mk)
    finally:
        sc.CASES['default_ssh_only'] = saved
    assert host_engine.lib.calls.count('od_step_oceandrift') == sc.STEPS
    for k in ('ID', 'lon', 'lat', 'z'):
        assert np.array_equal(np.asarray(getattr(o1.elements, k)), np.asarray(getattr(o2.elements, k)))
    for k in ('lon', 'lat', 'z', 'status'):
        assert np.array_equal(np.array(o1.history[k]), np.array(o2.history[k]), equal_nan=True)


def test_distributed_runs_refuse_the_correction(host_engine):
    from opendrift_b200.models.oceandrift import OceanDrift

    class _Dist:
        pass
    host_engine.dist = _Dist()
    o = OceanDrift(loglevel=50)
    o.set_config('drift:vertical_advection_correction', True)
    o.seed_elements(lon=3.0, lat=56.5, number=3, time=sc.common.Fixture('rk4_3d').start)
    with pytest.raises(NotImplementedError, match='vertical_advection_correction'):
        o.run(steps=1, time_step=600)


# -- the per-element functions against the reference's expressions --------------------------------------------------------------
def _ref_store(present, ids, age, dt, id_base, store):
    """update_previous_state (:645-657) literally: positional writes of the newly seeded, gather by ID, store by ID."""
    store = store.copy()
    if age is not None:
        rel = np.where(age == dt)[0]
        rel = rel[rel < len(store)]
        store[rel] = present[rel]
    k = ids.astype(np.int64) - id_base
    prev = store[k]
    store[k] = present
    return prev, store


def _ref_vadv(z, w, ssh, prev, floor, moving, at_surface, dt):
    """oceandrift.py:325-350 with the correction, NumPy 2 dtypes."""
    z = z.copy()
    app = np.where(z <= 0)[0] if at_surface else np.where(z < 0)[0]
    if len(app):
        fl = floor if isinstance(floor, np.ndarray) else np.full(len(z), floor, dtype=np.float32)
        wa = w[app]
        with np.errstate(invalid='ignore'):
            delta_zeta = ssh[app] - prev[app]
            w_surface = delta_zeta / dt
            total_depth = ssh[app] + fl[app]
            w_elevation = w_surface * (z[app] + total_depth) / total_depth
            wa = wa - w_elevation
            z[app] = np.minimum(0, z[app] + moving[app] * wa * dt)
    return z


@pytest.mark.parametrize('seed', range(6))
def test_corrected_vertical_advection_equals_numpy(seed):
    eng = sealevel_host.host_engine()
    rng = np.random.default_rng(seed)
    n = 5000
    for zdt in (np.float32, np.float64):
        for at_surface in (False, True):
            for dt in (600.0, -900.0, 60.0):
                z = (-rng.random(n) * 50).astype(zdt)
                z[:200] = 0
                z[200:300] = rng.random(100)                    # above the surface: untouched
                w = (rng.standard_normal(n) * 1e-3).astype(np.float32)
                ssh = (rng.standard_normal(n) * 0.7).astype(np.float32)
                ssh[300:400] = -np.abs(ssh[300:400]) - 1.5          # negative sea surface height
                prev = (ssh + rng.standard_normal(n).astype(np.float32) * 0.05).astype(np.float32)
                prev[400:450] = np.nan                              # no previous value (the reference's quirk)
                ssh[450:470] = np.nan
                moving = rng.integers(0, 2, n).astype(np.int32)
                for floor in ((5 + rng.random(n) * 80).astype(np.float32), 10000.0):
                    want = _ref_vadv(z, w, ssh, prev, floor, moving, at_surface, dt)
                    zt = torch.from_numpy(z.copy())
                    ft = torch.from_numpy(floor) if isinstance(floor, np.ndarray) else floor
                    eng.vertical_advection_corrected(zt, torch.from_numpy(w), torch.from_numpy(ssh), torch.from_numpy(prev), ft,
                                                     torch.from_numpy(moving), at_surface, dt)
                    got = zt.numpy()
                    assert got.dtype == want.dtype
                    assert np.array_equal(got, want, equal_nan=True)
                    assert np.isnan(got).any()


@pytest.mark.parametrize('seed', range(6))
def test_previous_store_equals_the_reference_sequence(seed):
    eng = sealevel_host.host_engine()
    rng = np.random.default_rng(seed)
    n_total = 3000
    for age_dt in (np.float32, np.float64):
        for dt in (600.0, -600.0):
            store = np.full(n_total, np.nan, dtype=np.float32)
            keep = rng.random(n_total) < 0.5
            store[keep] = rng.standard_normal(int(keep.sum())).astype(np.float32)
            alive = np.sort(rng.choice(n_total, 1800, replace=False))       # elements removed before this step
            ids = alive.astype(np.int32)
            n = len(ids)
            present = rng.standard_normal(n).astype(np.float32)
            age = (np.abs(dt) * rng.integers(1, 5, n) * np.sign(dt)).astype(age_dt)
            age[-300:] = dt                                                  # released this step
            for a in (age, None):
                want_prev, want_store = _ref_store(present, ids, a, dt, 0, store)
                st = torch.from_numpy(store.copy())
                prev = eng.store_previous_env(torch.from_numpy(present), torch.from_numpy(ids),
                                              None if a is None else torch.from_numpy(a), dt, 0, st)
                assert np.array_equal(prev.numpy(), want_prev, equal_nan=True)
                assert np.array_equal(st.numpy(), want_store, equal_nan=True)
                if a is not None:       # the quirk happened: some element gathered a value that is not its own stored one
                    assert not np.array_equal(want_prev, store[ids], equal_nan=True)
    # a shard: slots keyed by ID - id_base
    store = np.full(10, np.nan, dtype=np.float32)
    ids = np.arange(100, 110, dtype=np.int32)
    present = np.arange(10, dtype=np.float32)
    st = torch.from_numpy(store.copy())
    prev = eng.store_previous_env(torch.from_numpy(present), torch.from_numpy(ids), None, 600.0, 100, st)
    assert np.isnan(prev.numpy()).all() and np.array_equal(st.numpy(), present)


def test_environment_previous_follows_the_cell_sort(host_engine):
    """Enough elements for the cell sort, with the device generator: the arrays are re-ordered every step after the previous-step
    store ran.  What a subclass's update() reads from environment_previous.sea_surface_height, element by element, and the result
    equal those of the same run without the sort -- release in two batches and removal in between included (the store's quirk).
    With a sea-floor reader the step's environment is sampled before the lift and must follow the sort rather than be sampled
    again at the lifted depths."""
    import common
    from datetime import timedelta
    from opendrift_b200.models.oceandrift import OceanDrift
    from opendrift_b200.readers import reader_regular_grid

    class Recorder(OceanDrift):
        def update(self):
            self.rec.append((np.array(self.elements.ID, dtype=np.int64),
                             np.array(self.environment_previous.sea_surface_height, dtype=np.float32)))
            super().update()

    sorts = []
    plain_sort = host_engine.sort_by_cell

    def counting_sort(*a, **k):
        sorts.append(1)
        return plain_sort(*a, **k)
    host_engine.sort_by_cell = counting_sort

    def run(sort_every):
        fx = common.Fixture('rk4_3d_full')
        floor, ssh = sc.fields(fx)
        mk = lambda f, name, z=None: reader_regular_grid.Reader(fx.grid_lon, fx.grid_lat, z, fx.times, f, name=name)  # noqa: E731
        o = Recorder(loglevel=50)
        o.rec = []
        o.add_reader(mk({common.CUR[0]: fx.u, common.CUR[1]: fx.v, 'upward_sea_water_velocity': (20 * fx.w).astype(np.float32)},
                        'current', fx.grid_z))
        o.add_reader(mk({'sea_floor_depth_below_sea_level': np.repeat(floor[None], len(fx.times), axis=0)}, 'floor'))
        o.add_reader(mk({'sea_surface_height': ssh}, 'ssh'))
        for k, v in {'general:use_auto_landmask': False, 'environment:constant:land_binary_mask': 0, 'seed:ocean_only': False,
                     'drift:vertical_advection_correction': True, 'drift:advection_scheme': 'runge-kutta4', 'gpu:rng': 'philox',
                     'drift:deactivate_east_of': 3.6, 'gpu:sort_interval_steps': sort_every}.items():
            o.set_config(k, v)
        rng = np.random.default_rng(7)
        for n, t in ((150000, fx.start), (30000, fx.start + timedelta(seconds=2 * fx.dt))):
            o.seed_elements(lon=rng.uniform(2.3, 3.7, n), lat=rng.uniform(56.2, 56.9, n), z=-rng.uniform(0, 40, n).astype(np.float32),
                            time=t)
        o.run(steps=4, time_step=fx.dt, time_step_output=fx.dt)
        return o

    o0 = run(0)
    assert not sorts
    o1 = run(1)
    assert len(sorts) >= 3
    assert len(o0.rec) == len(o1.rec) == 4
    quirk = False
    for (i0, p0), (i1, p1) in zip(o0.rec, o1.rec):
        a, b = np.argsort(i0), np.argsort(i1)
        assert np.array_equal(i0[a], i1[b])
        assert np.array_equal(p0[a], p1[b], equal_nan=True)
        quirk |= bool(np.isnan(p0).any())
    assert quirk
    for el in ('elements', 'elements_deactivated'):
        e0, e1 = getattr(o0, el), getattr(o1, el)
        a, b = np.argsort(np.asarray(e0.ID)), np.argsort(np.asarray(e1.ID))
        for k in ('ID', 'lon', 'lat', 'z', 'status'):
            assert np.array_equal(np.asarray(getattr(e0, k))[a], np.asarray(getattr(e1, k))[b], equal_nan=True), (el, k)
