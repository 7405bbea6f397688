"""Per-step time (CUDA events) of OceanDrift with 5 M elements: u/v/w + sea floor + sea surface height + diffusivity readers,
vertical mixing and drift:vertical_advection_correction; and the same run without the sea surface height reader.  Prints one
JSON line with the card's name and power limit.  Run from the repository root: python tools/sealevel_timing.py"""
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
import sealevelcases as sc  # noqa: E402
from opendrift_b200.models.oceandrift import OceanDrift  # noqa: E402
from opendrift_b200.readers import reader_regular_grid  # noqa: E402

N, WARM, STEPS = 5_000_000, 3, 12


def run(with_ssh):
    fx = common.Fixture('rk4_3d_full')
    floor, ssh = sc.fields(fx)
    mk = lambda f, name, z=None: reader_regular_grid.Reader(fx.grid_lon, fx.grid_lat, z, fx.times, f, name=name)  # noqa: E731
    o = OceanDrift(loglevel=50)
    o.add_reader(mk({common.CUR[0]: fx.u, common.CUR[1]: fx.v, 'upward_sea_water_velocity': (20 * fx.w).astype(np.float32),
                     'ocean_vertical_diffusivity': common.Fixture('rk4_3d_mixing').kdiff}, 'current', fx.grid_z))
    o.add_reader(mk({'sea_floor_depth_below_sea_level': np.repeat(floor[None], len(fx.times), axis=0)}, 'floor'))
    if with_ssh:
        o.add_reader(mk({'sea_surface_height': ssh}, 'ssh'))
    for k, v in {'general:use_auto_landmask': False, 'environment:constant:land_binary_mask': 0, 'seed:ocean_only': False,
                 'drift:vertical_mixing': True, 'drift:vertical_advection_correction': True, 'gpu:rng': 'philox',
                 'drift:advection_scheme': 'runge-kutta4'}.items():
        o.set_config(k, v)
    rng = np.random.default_rng(0)
    lon = rng.uniform(2.3, 3.7, N)
    lat = rng.uniform(56.2, 56.9, N)
    z = -rng.uniform(0, 40, N).astype(np.float32)
    o.seed_elements(lon=lon, lat=lat, z=z, time=fx.start, terminal_velocity=-0.001)
    ev = []
    orig = o.release_elements

    def mark():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        ev.append(e)
        return orig()
    o.release_elements = mark
    o.run(steps=WARM + STEPS + 1, time_step=300, time_step_output=1200)
    torch.cuda.synchronize()
    per = ev[WARM].elapsed_time(ev[WARM + STEPS]) / STEPS
    return per, o.num_elements_active()


if __name__ == '__main__':
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    out = {'gpu': smi}
    for tag, ws in (('with_ssh_reader', True), ('without_ssh_reader', False), ('with_ssh_reader_again', True)):
        per, act = run(ws)
        out[tag] = {'ms_per_step': round(per, 3), 'active': act}
    print(json.dumps(out))
