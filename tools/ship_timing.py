"""Per-step time (CUDA events) of ShipDrift.run() at 10^6 and 10^7 ships (time_step 900 s, current and wind readers, a wave reader
with Hs and Tm02, the default diffusivity of 100 m^2/s with the device generator), against the reference's update() on the same
class -- what a user gets today by pasting the reference's ShipDrift onto the drop-in classes: the environment and element arrays
copied to the host, the spectrum and scipy's LinearNDInterpolator in NumPy.  The reference's body is timed for one step at 10^5
ships only: it is linear in the number of ships, and one step at 10^6 takes minutes.  Prints one JSON line with the card's name and power limit.  Needs the reference package that
oracle/build_ref.py copies to oracle/_ref (for the pasted update() and wforce.dat).  Run from the repository root:
python tools/ship_timing.py"""
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
import shipcases as sc  # noqa: E402
from opendrift_b200.models.shipdrift import ShipDrift  # noqa: E402
from opendrift_b200.readers import reader_regular_grid  # noqa: E402


def run(n, ref_update=None, warm=1, steps=3):
    fx = common.Fixture('rk4_3d_full')
    hs, tm, _, _, _, _ = sc.fields(fx)
    mk = lambda f, name, z=None, lon=fx.grid_lon, lat=fx.grid_lat: reader_regular_grid.Reader(lon, lat, z, fx.times, f,  # noqa: E731
                                                                                              name=name)
    Model = ShipDrift if ref_update is None else type('PastedShipDrift', (ShipDrift,), {'update': ref_update})
    o = Model(loglevel=50, wforce=sc.wforce_path())
    o.add_reader(mk({common.CUR[0]: fx.u, common.CUR[1]: fx.v}, 'current', fx.grid_z))
    o.add_reader(mk({'x_wind': fx.x_wind, 'y_wind': fx.y_wind}, 'wind', lon=fx.wind_lon, lat=fx.wind_lat))
    o.add_reader(mk({'sea_surface_wave_significant_height': hs, sc.TM02: tm}, 'waves'))
    for k, v in {'general:use_auto_landmask': False, 'environment:constant:land_binary_mask': 0, 'seed:ocean_only': False,
                 'gpu:rng': 'philox'}.items():
        o.set_config(k, v)
    rng = np.random.default_rng(0)
    kw = {k: np.resize(v, n) for k, v in sc.sizes('mixed', 1000).items()}
    o.seed_elements(lon=rng.uniform(2.3, 3.7, n), lat=rng.uniform(56.2, 56.9, n), time=fx.start, number=n, **kw)
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
    from opendrift.models.shipdrift import ShipDrift as RefShip
    for rnd in (1, 2):
        for n in (1_000_000, 10_000_000):
            out['shipdrift_%d_%d' % (n, rnd)] = {'ms_per_step': round(run(n), 2)}
            print(json.dumps(out), flush=True)
    out['reference_update_100000'] = {'ms_per_step': round(run(100_000, RefShip.update, warm=0, steps=1), 1)}
    print(json.dumps(out), flush=True)
