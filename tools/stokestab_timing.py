"""Per-step time (CUDA events) of OceanDrift with 5 M elements, cfg 4-like (u/v/w and diffusivity readers, a wind reader, RK4,
vertical mixing, the Phillips Stokes profile): the Stokes drift from a reader, against drift:use_tabularised_stokes_drift with no
Stokes reader (the Stokes drift and Hs parameterised from the wind every step).  Prints one JSON line with the card's name and
power limit.  Run from the repository root: python tools/stokestab_timing.py"""
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
import stokestabcases as sc  # noqa: E402
from opendrift_b200.models.oceandrift import OceanDrift  # noqa: E402
from opendrift_b200.readers import reader_regular_grid  # noqa: E402

N, WARM, STEPS = 5_000_000, 3, 12


def run(tabularised):
    fx = common.Fixture('rk4_3d_full')
    pos_x, pos_y, _, _, _ = sc.fields(fx)
    mk = lambda f, name, z=None, lon=fx.grid_lon, lat=fx.grid_lat: reader_regular_grid.Reader(lon, lat, z, fx.times, f,  # noqa: E731
                                                                                              name=name)
    o = OceanDrift(loglevel=50)
    o.add_reader(mk({common.CUR[0]: fx.u, common.CUR[1]: fx.v, 'upward_sea_water_velocity': (20 * fx.w).astype(np.float32),
                     'ocean_vertical_diffusivity': common.Fixture('rk4_3d_mixing').kdiff}, 'current', fx.grid_z))
    o.add_reader(mk({'x_wind': fx.x_wind, 'y_wind': fx.y_wind}, 'wind', lon=fx.wind_lon, lat=fx.wind_lat))
    if not tabularised:
        o.add_reader(mk({sc.SX: pos_x, sc.SY: pos_y}, 'stokes'))
    for k, v in {'general:use_auto_landmask': False, 'environment:constant:land_binary_mask': 0, 'seed:ocean_only': False,
                 'drift:vertical_mixing': True, 'gpu:rng': 'philox', 'drift:advection_scheme': 'runge-kutta4',
                 'drift:stokes_drift_profile': 'Phillips', 'drift:use_tabularised_stokes_drift': tabularised}.items():
        o.set_config(k, v)
    rng = np.random.default_rng(0)
    lon = rng.uniform(2.3, 3.7, N)
    lat = rng.uniform(56.2, 56.9, N)
    z = -rng.uniform(0, 40, N).astype(np.float32)
    o.seed_elements(lon=lon, lat=lat, z=z, time=fx.start)
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
    for tag, tab in (('stokes_reader', False), ('tabularised', True), ('stokes_reader_again', False), ('tabularised_again', True)):
        per, act = run(tab)
        out[tag] = {'ms_per_step': round(per, 3), 'active': act}
    print(json.dumps(out))
