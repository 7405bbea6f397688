"""drift:use_tabularised_stokes_drift (tests/stokestabcases.py) on the host build of the device sources: the drop-in OceanDrift
against runs of the unmodified reference, positions and the values of the public get_environment; the per-element function of
csrc/od_stokes.cuh against the reference's NumPy expressions restated here; and the refusal in distributed runs."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import common
import stokestabcases as sc
import stokestab_host
from opendrift_b200.models.environment import stokes_coefficients


@pytest.fixture()
def host_engine(monkeypatch):
    eng = stokestab_host.host_engine()
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    monkeypatch.setattr(E, 'default_engine', lambda device=None: eng)
    monkeypatch.setattr(B, 'default_engine', lambda device=None: eng)
    yield eng


@pytest.mark.parametrize('case', list(sc.CASES))
def test_tabularised_stokes_case_equals_the_reference(case, host_engine):
    o = sc.run_product(case)
    sc.check(o, case)
    calls = host_engine.lib.calls
    assert 'od_stokes_parameterised' in calls
    if case == 'fetch25000':         # the stock recipe keeps its fused step
        assert calls.count('od_step_oceandrift') == sc.STEPS
    if case == 'stokes_reader_positive':
        env = o.stokes_tab_env
        assert np.all(env[sc.SX] > 0)            # the reader's values, not the wind's
    if case == 'stokes_reader_nonpositive':
        ref = np.load(sc.GOLDEN)
        assert np.any(ref[case + '__env_' + sc.SX] > 0)


# -- the per-element function against the reference's expressions ---------------------------------------------------------------
def _ref_parameterised(xw, yw, fetch, masked=False):
    """wave_stokes_drift_parameterised / wave_significant_height_parameterised (physics_methods.py:488-568) literally, the results
    stored into float32 environment fields.  The reference's environment holds masked arrays, which np.ma.power squares in float64
    (masked=True); for a non-finite wind np.ma also masks the result and keeps the input, which the device does not reproduce:
    there the plain float64 expressions (masked=False) are the rule (NaN stays NaN, an infinite speed is capped at 30)."""
    cw, ch = stokes_coefficients(fetch)
    if masked:
        xw, yw = np.ma.array(xw), np.ma.array(yw)
        sq = lambda a: a ** 2                                                        # noqa: E731
    else:
        sq = lambda a: a.astype(np.float64) ** 2                                     # noqa: E731
    with np.errstate(invalid='ignore', over='ignore'):
        ws = np.sqrt(sq(xw) + sq(yw))
        ws[ws > 30] = 30
        wf = np.polyval(cw, ws)
        us, vs = np.asarray((xw * wf).astype(np.float32)), np.asarray((yw * wf).astype(np.float32))
        hs = np.asarray(np.polyval(ch, ws).astype(np.float32))
    return us, vs, hs


def _winds(seed, n):
    rng = np.random.default_rng(seed)
    xw = (rng.standard_normal(n) * 12).astype(np.float32)
    yw = (rng.standard_normal(n) * 12).astype(np.float32)
    sub = np.float32(1e-40)
    special = [(np.nan, 1.0), (1.0, np.nan), (0.0, 0.0), (-0.0, -0.0), (-0.0, 0.0), (sub, -sub), (30.0, 0.0), (0.0, -30.0),
               (18.0, 24.0), (np.float32(30.000002), 0.0), (29.999998, 0.0), (45.0, -10.0), (np.inf, 0.0), (-np.inf, 3.0),
               (1e-20, 1e-20), (3e19, 0.0)]
    for k, (a, b) in enumerate(special[:n]):
        xw[k], yw[k] = a, b
    return xw, yw


@pytest.mark.parametrize('fetch', ['5000', '25000', '50000'])
def test_parameterisation_equals_numpy(fetch):
    eng = stokestab_host.host_engine()
    cw, ch = stokes_coefficients(fetch)
    assert len(cw) == {'5000': 4, '25000': 7, '50000': 7}[fetch] and len(ch) == 2
    for seed in range(4):
        xw, yw = _winds(seed, 20000)
        want = _ref_parameterised(xw, yw, fetch)
        fin = np.isfinite(xw) & np.isfinite(yw)
        for w, m in zip(want, _ref_parameterised(xw[fin], yw[fin], fetch, masked=True)):
            assert np.array_equal(w[fin], m)
        t = lambda a: torch.from_numpy(a)         # noqa: E731
        us, vs, hs = (torch.full((len(xw),), 7.0, dtype=torch.float32) for _ in range(3))
        eng.stokes_parameterised(t(xw), t(yw), cw, ch, us, vs, hs)
        for got, w in zip((us, vs, hs), want):
            assert np.array_equal(got.numpy(), w, equal_nan=True)
            assert np.array_equal(np.signbit(got.numpy()), np.signbit(w))
        # one output only: the other is not written
        us2, vs2, hs2 = (torch.full((len(xw),), 7.0, dtype=torch.float32) for _ in range(3))
        eng.stokes_parameterised(t(xw), t(yw), cw, ch, us2, vs2, None)
        eng.stokes_parameterised(t(xw), t(yw), cw, ch, None, None, hs2)
        assert np.array_equal(us2.numpy(), want[0], equal_nan=True) and np.array_equal(hs2.numpy(), want[2], equal_nan=True)
    assert np.isnan(want[0]).any() and np.isinf(want[0]).any()


def test_stokes_drift_off_gives_the_parameterised_environment(host_engine):
    """drift:stokes_drift = False: the step's environment has no Stokes variables (the reference stops there, with no field to
    write the parameterised drift into).  The run goes on and moves the elements exactly as without the option, and the public
    get_environment, asked for the Stokes variables, returns the values parameterised from the wind it returns."""
    runs = []
    for tab in (True, False):
        o = sc.run_product('fetch25000', extra_config={'drift:stokes_drift': False, 'drift:use_tabularised_stokes_drift': tab})
        runs.append(o)
    a, b = runs
    for k in ('ID', 'lon', 'lat', 'z'):
        assert np.array_equal(np.asarray(getattr(a.elements, k)), np.asarray(getattr(b.elements, k)))
    env = a.stokes_tab_env
    us, vs, hs = _ref_parameterised(env['x_wind'], env['y_wind'], '25000', masked=True)
    assert np.array_equal(env[sc.SX], us) and np.array_equal(env[sc.SY], vs) and np.array_equal(env[sc.HS], hs)
    assert np.abs(us).max() > 0.01
    assert np.all(b.stokes_tab_env[sc.SX] == 0)


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
    import stokestab_host as sh
    import stokestabcases as cases
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    eng = sh.host_engine()
    E.default_engine = B.default_engine = lambda device=None: eng
    try:
        cases.run_product('fetch25000', extra_config={'gpu:rng': 'philox'})
        q.put((rank, 'ran', ''))
    except NotImplementedError as e:
        q.put((rank, 'refused', str(e)))
    dist.destroy_process_group()


def test_two_rank_run_refuses_the_tabularised_stokes_drift():
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
    assert all('drift:use_tabularised_stokes_drift' in r[2] for r in res)
