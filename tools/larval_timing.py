"""Per-step time (CUDA events) of LarvalFish.run() at 10^6 and 5*10^6 elements with time_step 3600 s and the default
vertical_mixing:timestep of 60 s (60 inner mixing iterations), T and S readers, a diffusivity profile on the current's reader and the
device generator, against the reference's LarvalFish class body pasted onto the drop-in OceanDrift -- what a user gets without this
model: one mixing launch per inner iteration with the terminal velocity recomputed in NumPy on host copies between them, and the
hatching, growth and migration in NumPy.  The pasted body is timed at 10^5 elements.  Prints one JSON line with the card's name and
power limit.  Needs the reference package that oracle/build_ref.py copies to oracle/_ref (for the pasted body).  Run from the
repository root: python tools/larval_timing.py"""
import json
import os
import subprocess
import sys
from datetime import timedelta

import numpy as np
import torch

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, _ROOT)
sys.path.insert(0, os.path.join(_ROOT, 'tests'))
import common  # noqa: E402
import larvalcases  # noqa: E402
from opendrift_b200.models.larvalfish import LarvalFish, LarvalFishElement  # noqa: E402
from opendrift_b200.models.oceandrift import OceanDrift  # noqa: E402
from opendrift_b200.readers import reader_regular_grid  # noqa: E402


def pasted_class(ref):
    """The reference's LarvalFish class body on the drop-in OceanDrift."""
    body = {k: v for k, v in vars(ref).items() if callable(v) and k != '__init__'}
    body['ElementType'] = LarvalFishElement
    body['required_variables'] = ref.required_variables

    def init(self, *a, **kw):
        OceanDrift.__init__(self, *a, **kw)
        self._add_config({'IBM:fraction_of_timestep_swimming': {'type': 'float', 'default': 0.15, 'min': 0.0, 'max': 1.0,
                                                                'units': 'fraction', 'description': '', 'level': 3}})
        for k in ('drift:vertical_mixing', 'drift:vertical_mixing_at_surface', 'drift:vertical_advection_at_surface'):
            self._set_config_default(k, True)
    body['__init__'] = init
    return type('PastedLarvalFish', (OceanDrift,), body)


def run(n, Model, warm=1, steps=3):
    fx = common.Fixture('rk4_3d_full')
    times = [fx.start + timedelta(hours=k) for k in range(8)]
    mk = lambda f, name, z=None: reader_regular_grid.Reader(fx.grid_lon, fx.grid_lat, z, times, f, name=name)      # noqa: E731
    temp, salt = larvalcases.fields(fx)[:2]
    pad = lambda a: np.concatenate([a, np.repeat(a[-1:], len(times) - len(a), axis=0)])                         # noqa: E731
    k = np.maximum(common.Fixture('rk4_3d_mixing').kdiff, np.float32(0.02))
    o = Model(loglevel=50)
    o.add_reader(mk({common.CUR[0]: pad(fx.u), common.CUR[1]: pad(fx.v), 'ocean_vertical_diffusivity': pad(k)}, 'current', fx.grid_z))
    o.add_reader(mk({'sea_water_temperature': pad(temp), 'sea_water_salinity': pad(salt)}, 'ts'))
    for key, v in {'general:use_auto_landmask': False, 'environment:constant:land_binary_mask': 0, 'seed:ocean_only': False,
                   'gpu:rng': 'philox', 'vertical_mixing:diffusivitymodel': 'environment'}.items():
        o.set_config(key, v)
    rng = np.random.default_rng(0)
    o.seed_elements(lon=rng.uniform(2.3, 3.7, n), lat=rng.uniform(56.2, 56.9, n), time=fx.start, number=n,
                    z=-rng.uniform(5, 20, n).astype(np.float32), hatched=(np.arange(n) % 2).astype(np.uint8),
                    stage_fraction=rng.uniform(0.9, 1.0, n).astype(np.float32))
    ev = []
    orig = o.release_elements

    def mark():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        ev.append(e)
        return orig()
    o.release_elements = mark
    o.run(steps=warm + steps + 1, time_step=3600, time_step_output=3600)
    torch.cuda.synchronize()
    return ev[warm].elapsed_time(ev[warm + steps]) / steps


if __name__ == '__main__':
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    out = {'gpu': smi}
    from oracle import refrun
    refrun.setup()
    from opendrift.models.larvalfish import LarvalFish as RefLarval
    for rnd in (1, 2):
        for n in (1_000_000, 5_000_000):
            out['larvalfish_%d_%d' % (n, rnd)] = {'ms_per_step': round(run(n, LarvalFish), 2)}
            print(json.dumps(out), flush=True)
    out['reference_body_on_oceandrift_100000'] = {'ms_per_step': round(run(100_000, pasted_class(RefLarval), warm=1, steps=2), 1)}
    print(json.dumps(out), flush=True)
