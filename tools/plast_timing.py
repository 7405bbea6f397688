"""Per-step time (CUDA events) of PlastDrift.run() at 10^6 and 10^7 elements with vertical_mixing:mixingmodel = 'analytical' and
'randomwalk' (time_step 900 s, current and wind readers, the defaults otherwise: tabularised Stokes drift from the wind, Sundby 1983
for the random walk with its 15 inner iterations, the device generator), against the reference's PlastDrift.update and
update_particle_depth pasted onto the drop-in classes -- what a user gets today: the depth drawn in NumPy on host copies of the
environment and element arrays, then the Stokes and wind helpers.  The pasted body is timed at 10^5 elements with the legacy generator.
Prints one JSON line with the card's name and power limit.  Needs the reference package that oracle/build_ref.py copies to
oracle/_ref (for the pasted body).  Run from the repository root: python tools/plast_timing.py"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, 'tests'))
import common  # noqa: E402
from opendrift_b200.models.plastdrift import PlastDrift  # noqa: E402
from opendrift_b200.readers import reader_regular_grid  # noqa: E402


def run(n, model, pasted=None, warm=1, steps=3):
    fx = common.Fixture('rk4_3d_full')
    mk = lambda f, name, z=None, lon=fx.grid_lon, lat=fx.grid_lat: reader_regular_grid.Reader(lon, lat, z, fx.times, f,  # noqa: E731
                                                                                              name=name)
    Model = PlastDrift if pasted is None else type('PastedPlastDrift', (PlastDrift,), {
        'update': pasted.update, 'update_particle_depth': pasted.update_particle_depth})
    o = Model(loglevel=50)
    o.add_reader(mk({common.CUR[0]: fx.u, common.CUR[1]: fx.v}, 'current', fx.grid_z))
    o.add_reader(mk({'x_wind': fx.x_wind, 'y_wind': fx.y_wind}, 'wind', lon=fx.wind_lon, lat=fx.wind_lat))
    for k, v in {'general:use_auto_landmask': False, 'environment:constant:land_binary_mask': 0, 'seed:ocean_only': False,
                 'gpu:rng': 'philox' if pasted is None else 'numpy', 'vertical_mixing:mixingmodel': model}.items():
        o.set_config(k, v)
    rng = np.random.default_rng(0)
    o.seed_elements(lon=rng.uniform(2.3, 3.7, n), lat=rng.uniform(56.2, 56.9, n), time=fx.start, number=n,
                    z=-rng.uniform(0, 20, n).astype(np.float32))
    ev = []
    orig = o.release_elements

    def mark():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        ev.append(e)
        return orig()
    o.release_elements = mark
    o.run(steps=warm + steps + 1, time_step=900, time_step_output=900)
    torch.cuda.synchronize()
    return ev[warm].elapsed_time(ev[warm + steps]) / steps


if __name__ == '__main__':
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    out = {'gpu': smi}
    from oracle import refrun
    refrun.setup()
    from opendrift.models.plastdrift import PlastDrift as RefPlast
    for rnd in (1, 2):
        for model in ('analytical', 'randomwalk'):
            for n in (1_000_000, 10_000_000):
                out['%s_%d_%d' % (model, n, rnd)] = {'ms_per_step': round(run(n, model), 2)}
                print(json.dumps(out), flush=True)
    out['reference_update_analytical_100000'] = {'ms_per_step': round(run(100_000, 'analytical', RefPlast, warm=1, steps=2), 1)}
    print(json.dumps(out), flush=True)
