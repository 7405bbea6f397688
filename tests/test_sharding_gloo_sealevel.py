"""World-size-2 runs (gloo, CPU, host engine) with a varying sea surface height: index shards with sea floor, sea surface height
and diffusivity readers and vertical mixing equal the unsharded run bit for bit; drift:vertical_advection_correction is refused in
distributed runs (the reference's previous-step store depends on positions in the whole element array)."""
import os
import socket
import sys

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp

import common

# draws keyed by element ID (gpu:rng = philox): the legacy generator's draws are per process
_CFG = {'gpu:rng': 'philox'}


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(case):
    import sealevel_host
    import sealevelcases as sc
    import opendrift_b200.engine as E
    import opendrift_b200.models.basemodel as B
    eng = sealevel_host.host_engine()
    E.default_engine = B.default_engine = lambda device=None: eng
    try:
        o = sc.run_product(case, extra_config=_CFG)
    except NotImplementedError as e:
        return None, str(e)
    return o, sc.summary(o)


def _worker(rank, world, port, q, case):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    sys.path.insert(0, common.ROOT)
    sys.path.insert(0, os.path.join(common.ROOT, 'tests'))
    o, s = _run(case)
    if o is None:
        q.put((rank, 'refused', s))
    else:
        q.put((rank, o.shard, s['id'], s['lon'], s['lat'], s['z'], s['d_id'], s['d_z'], [str(c) for c in s['cats']],
               s['d_status']))
    dist.destroy_process_group()


def _two_ranks(case):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, case)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in procs], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
    return res


def test_two_rank_run_with_sea_level_and_mixing_equals_the_unsharded_run():
    res = _two_ranks('mixing')
    _, s = _run('mixing')
    ids = np.concatenate([r[2] for r in res])
    assert len(ids) == len(s['id']) and len(ids) > 0
    o, ro = np.argsort(ids), np.argsort(s['id'])
    assert np.array_equal(ids[o], s['id'][ro])
    for k, j in (('lon', 3), ('lat', 4), ('z', 5)):
        assert np.array_equal(np.concatenate([r[j] for r in res])[o], s[k][ro]), k
    assert sum(len(r[6]) for r in res) == len(s['d_id'])


def test_two_rank_run_refuses_the_vertical_advection_correction():
    res = _two_ranks('correction_rk4')
    assert [r[1] for r in res] == ['refused', 'refused']
    assert all('vertical_advection_correction' in r[2] for r in res)
