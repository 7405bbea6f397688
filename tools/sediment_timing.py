"""Per-step time (CUDA events) of SedimentDrift.run() at 10^6 and 5*10^6 elements (time_step 1800 s, vertical_mixing:timestep 60 s:
30 inner iterations, Large et al. 1994 diffusivity from a wind reader, a current reader, the resuspension example's 30 m fallback
floor, the device generator), against the same model written as a subclass of the drop-in OceanDrift -- update() in SedimentDrift's
order, bottom_interaction and resuspension on NumPy arrays -- which takes the per-iteration mixing path (one launch, a copy of z to
the host and the hook per inner iteration).  The two alternate, twice per size.  Prints one JSON line with the card's name and power
limit.  Run from the repository root: python tools/sediment_timing.py"""
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
from opendrift_b200.models.oceandrift import OceanDrift  # noqa: E402
from opendrift_b200.models.sedimentdrift import SedimentDrift  # noqa: E402
from opendrift_b200.readers import reader_regular_grid  # noqa: E402

WARM, STEPS = 1, 3


class HostSettling(OceanDrift):
    """SedimentDrift's recipe on OceanDrift, with its two rules on host arrays."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self._add_config({'vertical_mixing:resuspension_threshold': {'type': 'float', 'default': 0.2, 'min': 0, 'max': 3,
                                                                     'units': 'm/s', 'description': 'resuspension threshold', 'level': 1}})

    def update(self):
        self.advect_ocean_current()
        self.vertical_advection()
        self.advect_wind()
        self.stokes_drift()
        self.vertical_mixing()
        self.resuspension()

    def bottom_interaction(self, seafloor_depth):
        el = self.elements
        el.moving[(el.z <= seafloor_depth) & (el.moving == 1)] = 0

    def resuspension(self):
        el, env = self.elements, self.environment
        speed = np.sqrt(env.x_sea_water_velocity ** 2 + env.y_sea_water_velocity ** 2)
        up = (speed > self.get_config('vertical_mixing:resuspension_threshold')) & (el.moving == 0)
        el.moving[up] = 1
        el.z[up] = el.z[up] + .01


def run(Model, n):
    fx = common.Fixture('rk4_3d_full')
    mk = lambda f, name, z=None, lon=fx.grid_lon, lat=fx.grid_lat: reader_regular_grid.Reader(lon, lat, z, fx.times, f,  # noqa: E731
                                                                                              name=name)
    o = Model(loglevel=50)
    o.add_reader(mk({common.CUR[0]: fx.u, common.CUR[1]: fx.v}, 'current', fx.grid_z))
    o.add_reader(mk({'x_wind': fx.x_wind, 'y_wind': fx.y_wind}, 'wind', lon=fx.wind_lon, lat=fx.wind_lat))
    for k, v in {'general:use_auto_landmask': False, 'environment:constant:land_binary_mask': 0, 'seed:ocean_only': False,
                 'drift:vertical_mixing': True, 'vertical_mixing:diffusivitymodel': 'windspeed_Large1994', 'gpu:rng': 'philox',
                 'environment:fallback:sea_floor_depth_below_sea_level': 30, 'vertical_mixing:resuspension_threshold': 0.5,
                 'vertical_mixing:timestep': 60}.items():
        o.set_config(k, v)
    rng = np.random.default_rng(0)
    o.seed_elements(lon=rng.uniform(2.3, 3.7, n), lat=rng.uniform(56.2, 56.9, n), z=-rng.uniform(0, 30, n).astype(np.float32),
                    terminal_velocity=np.float32(-0.01), time=fx.start)
    ev = []
    orig = o.release_elements

    def mark():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        ev.append(e)
        return orig()
    o.release_elements = mark
    o.run(steps=WARM + STEPS + 1, time_step=1800, time_step_output=1800)
    torch.cuda.synchronize()
    per = ev[WARM].elapsed_time(ev[WARM + STEPS]) / STEPS
    return per, int((np.asarray(o.elements.moving) == 0).sum())


if __name__ == '__main__':
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    out = {'gpu': smi}
    for n in (1_000_000, 5_000_000):
        for rnd in (1, 2):
            for tag, Model in (('sedimentdrift', SedimentDrift), ('per_iteration_hooks', HostSettling)):
                per, settled = run(Model, n)
                out['%s_%d_%d' % (tag, n, rnd)] = {'ms_per_step': round(per, 2), 'settled': settled}
    print(json.dumps(out))
