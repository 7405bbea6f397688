"""Kernel-alone timings of the bench's launches for one build of libodcuda.so (ODCUDA_LIB selects a tuning build):
fused RK4 + vertical advection (the bench's launch), current only, fast arithmetic -- CUDA events, 10 M cell-sorted
particles in the 512x512x50 u/v/w field; prints one JSON line incl. a checksum of the new positions so that builds that
must agree bit for bit can be compared."""
import hashlib
import json
import os
import sys
from datetime import timedelta

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opendrift_b200 import synthetic as syn          # noqa: E402
from opendrift_b200.engine import Engine             # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
eng = Engine(0)
g = syn.GridSpec()
times = syn.slab_times(3)
slabs = [tuple(torch.from_numpy(a).cuda() for a in syn.double_gyre_uv(g, (t - syn.T0).total_seconds())) for t in times]
w = torch.from_numpy(syn.upward_w(g)).cuda()
grp = eng.add_group(g.lon, g.lat, g.z, 2, times, lambda ti, c: slabs[ti][c], (0.0, 0.0))
wgrp = eng.add_group(g.lon, g.lat, g.z, 1, times, lambda ti, c: w, (0.0,))
lon0, lat0, z0 = syn.particle_cloud(n, seed=5)
lon, lat, z = eng.to_device(lon0.astype(np.float64)), eng.to_device(lat0.astype(np.float64)), eng.to_device(z0)
perm = eng.sort_by_cell(grp, lon, lat, z)
lon, lat, z = eng.permute(perm, lon), eng.permute(perm, lat), eng.permute(perm, z)
t, dt = times[0] + timedelta(seconds=300), timedelta(seconds=600)


def digest(*ts):
    # in the original particle order: the cell sort places particles within a cell by atomic counter, so the sorted order
    # differs between runs
    h = hashlib.sha1()
    for x in ts:
        h.update(eng.permute(perm, x, inverse=True).cpu().numpy().tobytes())
    return h.hexdigest()[:12]


def timeit(fn, reps=7):
    out, res = [], None
    for k in range(reps + 2):
        tl, ta, tz = lon.clone(), lat.clone(), z.clone()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn(tl, ta, tz)
        b.record()
        torch.cuda.synchronize()
        if k >= 2:
            out.append(a.elapsed_time(b))
        res = (tl, ta, tz)
    return float(np.median(out)), float(np.min(out)), digest(*res)


# clock ramp
r0 = torch.cuda.Event(enable_timing=True)
for _ in range(300):
    eng.step_oceandrift(grp, 'runge-kutta4', t, dt, lon.clone(), lat.clone(), z.clone(), w_group=wgrp)
torch.cuda.synchronize()
res = {'lib': os.environ.get('ODCUDA_LIB', 'default'), 'n': n}
def spec(on):
    if hasattr(eng, 'set_spec'):
        try:
            eng.set_spec(on)
        except Exception:
            pass


t1 = times[1]                      # a step that starts on a reader time (single-slab time mode at the first stage)
t5 = times[0] + timedelta(seconds=3000)      # a step that ends on a reader time (single-slab mode at the last stage)
for name, fn, sp in (
        ('fused', lambda a, b, c: eng.step_oceandrift(grp, 'runge-kutta4', t, dt, a, b, c, w_group=wgrp), True),
        ('fused_gen', lambda a, b, c: eng.step_oceandrift(grp, 'runge-kutta4', t, dt, a, b, c, w_group=wgrp), False),
        ('fused_t1', lambda a, b, c: eng.step_oceandrift(grp, 'runge-kutta4', t1, dt, a, b, c, w_group=wgrp), True),
        ('fused_t1_gen', lambda a, b, c: eng.step_oceandrift(grp, 'runge-kutta4', t1, dt, a, b, c, w_group=wgrp), False),
        ('fused_t5', lambda a, b, c: eng.step_oceandrift(grp, 'runge-kutta4', t5, dt, a, b, c, w_group=wgrp), True),
        ('fused_t5_gen', lambda a, b, c: eng.step_oceandrift(grp, 'runge-kutta4', t5, dt, a, b, c, w_group=wgrp), False),
        ('cur', lambda a, b, c: eng.advect_current(grp, 'runge-kutta4', t, dt, a, b, c), True),
        ('cur_gen', lambda a, b, c: eng.advect_current(grp, 'runge-kutta4', t, dt, a, b, c), False),
        ('fast', lambda a, b, c: eng.step_oceandrift(grp, 'runge-kutta4', t, dt, a, b, c, w_group=wgrp, fast=1), True)):
    spec(sp)
    try:
        med, mn, dg = timeit(fn)
        res[name + '_ms'], res[name + '_min_ms'], res[name + '_sha'] = round(med, 4), round(mn, 4), dg
    except Exception as ex:
        res[name + '_err'] = str(ex)[:80]
print(json.dumps(res))
