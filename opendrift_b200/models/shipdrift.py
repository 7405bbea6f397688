"""ShipDrift (ships adrift) on the GPU path: the reference's model class (opendrift/models/shipdrift.py) with the same element type
(ShipObject :32-78), required variables (:89-103), configuration, seeding of the drag coefficients (:157-214) and update() (:216-343),
the latter as ONE kernel launch per time step (od_ship_step, csrc/od_ship.cuh): current move, wind / wave / form-drag force balance,
ship move and stranding.

Before the launch, update() takes the reference's decisions over the whole element array (physics_methods.py:893-943,
shipdrift.py:302-311) from reductions on the device (od_minmax_f32): Hs from a reader or from the wind, the wave period from Tm02, Tp
or the wind (zeros replaced by the mean of the positive periods), and the wave direction from the wind or from the Stokes drift.

The wave force table: the reference reads wforce.dat from its own package directory.  Here it is `ShipDrift(wforce=<path>)`, or
models/wforce.dat of an installed `opendrift` package.  The table goes to the device once per model instance, with the tetrahedra of
the Delaunay triangulation that scipy's LinearNDInterpolator builds on it (the lookup is that interpolator's, bit for bit).
"""
import importlib.util
import logging
import os

import numpy as np

from ..config import CONFIG_LEVEL_ESSENTIAL, CONFIG_LEVEL_ADVANCED
from ..elements import LagrangianArray
from ..engine import SHIP_ELEMENTS
from .basemodel import OpenDriftSimulation

logger = logging.getLogger('opendrift_b200')

TM02 = 'sea_surface_wave_mean_period_from_variance_spectral_density_second_frequency_moment'
TP = 'sea_surface_wave_period_at_variance_spectral_density_maximum'
HS = 'sea_surface_wave_significant_height'
STOKES = ('sea_surface_wave_stokes_drift_x_velocity', 'sea_surface_wave_stokes_drift_y_velocity')


class ShipObject(LagrangianArray):
    """shipdrift.py:32-78"""
    variables = LagrangianArray.add_variables([
        ('orientation', {'dtype': np.uint8, 'units': '1', 'default': 1}),
        ('length', {'dtype': np.float32, 'units': 'm', 'min': 1, 'max': 500, 'description': 'Length of ship',
                    'level': CONFIG_LEVEL_ESSENTIAL, 'default': 80}),
        ('height', {'dtype': np.float32, 'units': 'm', 'min': 1, 'max': 100,
                    'description': 'Total height of ship (above and below waterline)', 'level': CONFIG_LEVEL_ESSENTIAL, 'default': 8}),
        ('draft', {'dtype': np.float32, 'units': 'm', 'min': 1, 'max': 30, 'description': 'Draft of ship (depth below water)',
                   'level': CONFIG_LEVEL_ESSENTIAL, 'default': 4.0}),
        ('beam', {'dtype': np.float32, 'min': 1, 'max': 70, 'units': 'm', 'description': 'Beam (width) of ship',
                  'level': CONFIG_LEVEL_ESSENTIAL, 'default': 10}),
        ('wind_drag_coeff', {'dtype': np.float32, 'units': '1', 'default': 1}),
        ('water_drag_coeff', {'dtype': np.float32, 'units': '1', 'default': 1}),
        ('jibeProbability', {'dtype': np.float32, 'units': '1/h', 'default': 0.04})])      # (not used by update())


def find_wforce():
    """models/wforce.dat of an installed `opendrift` package, located without importing it; None if there is none."""
    try:
        spec = importlib.util.find_spec('opendrift')
    except (ImportError, ValueError):
        return None
    for d in (spec.submodule_search_locations or []) if spec is not None else []:
        p = os.path.join(d, 'models', 'wforce.dat')
        if os.path.exists(p):
            return p
    return None


def read_wforce(path):
    """shipdrift.py:107-136, including its fill order F[o, i, :] = the i-th row of the block (i over the drafts)."""
    wf = {}
    with open(path, 'r') as w:
        w.readline()
        nbeam = int(w.readline().split()[0])
        wf['nbeam'] = nbeam
        wf['BL'] = np.array(w.readline().split()[0:nbeam], dtype=float)
        ndraft = int(w.readline().split()[0])
        wf['ndraft'] = ndraft
        wf['DL'] = np.array(w.readline().split()[0:ndraft], dtype=float)
        nomega = int(w.readline().split()[0])
        wf['nomega'] = nomega
        wf['omega'] = np.zeros((nomega))
        wf['F'] = np.zeros((nomega, nbeam, ndraft))
        wf['D'] = np.zeros((nomega, nbeam, ndraft))
        for o in range(nomega):
            wf['omega'][o] = float(w.readline().split()[0])
            for i in range(ndraft):
                wf['F'][o, i, :] = w.readline().split()[0:nbeam]
            for i in range(ndraft):
                wf['D'][o, i, :] = w.readline().split()[0:nbeam]
    return wf


def wforce_interpolators(wf):
    """The reference's two LinearNDInterpolator objects (shipdrift.py:137-145): same points, same order, same Qhull options."""
    import scipy.interpolate
    wi_omega, wi_BL, wi_DL = np.meshgrid(wf['omega'], wf['BL'], wf['DL'], indexing='ij')
    pts = (wi_omega.ravel(), wi_BL.ravel(), wi_DL.ravel())
    return (scipy.interpolate.LinearNDInterpolator(pts, wf['F'].ravel()),
            scipy.interpolate.LinearNDInterpolator(pts, wf['D'].ravel()))


def wforce_table(wf, ipF):
    """(wtab float64, wbox int32, (nomega, nbeam, ndraft)) for od_ship_step (layout in csrc/od_ship.cuh).  Every non-degenerate
    tetrahedron of the interpolator's triangulation lies in one grid box; a box lists its tetrahedra in the triangulation's order, so
    that the first one containing a query (barycentric coordinates >= -100 DBL_EPSILON) is the one scipy finds.  Degenerate (flat)
    tetrahedra have a NaN transform and never contain a point; they are left out."""
    tri = ipF.tri
    axes = (wf['omega'], wf['BL'], wf['DL'])
    dims = tuple(len(a) for a in axes)
    F, D = wf['F'].ravel(), wf['D'].ravel()
    nbox = (dims[0] - 1) * (dims[1] - 1) * (dims[2] - 1)
    per_box = [[] for _ in range(nbox)]
    for k in range(len(tri.simplices)):
        T = tri.transform[k]
        if np.isnan(T).any():
            continue
        v = tri.points[tri.simplices[k]]
        lo = [int(np.searchsorted(ax, v[:, j].min())) for j, ax in enumerate(axes)]
        hi = [int(np.searchsorted(ax, v[:, j].max())) for j, ax in enumerate(axes)]
        if any(h - l != 1 for l, h in zip(lo, hi)):
            raise ValueError('wforce table: a tetrahedron of the triangulation spans more than one grid box')
        per_box[(lo[0] * (dims[1] - 1) + lo[1]) * (dims[2] - 1) + lo[2]].append(k)
    rows, wbox = [], [0]
    for ks in per_box:
        for k in ks:
            s = tri.simplices[k]
            rows.append(np.concatenate([tri.transform[k, :3, :].ravel(), tri.transform[k, 3, :], F[s], D[s]]))
        wbox.append(len(rows))
    wtab = np.concatenate([axes[0], axes[1], axes[2], np.asarray(rows, dtype=np.float64).ravel()])
    return wtab.astype(np.float64), np.asarray(wbox, dtype=np.int32), dims


class ShipDrift(OpenDriftSimulation):
    """Ships adrift (shipdrift.py:80-343; Soergaard and Vada 1998)."""
    ElementType = ShipObject
    # general:coastline_action stays 'none' here; the reference's default is 'stranding' (against the GSHHG mask)
    _coast_reference_default = ('stranding', 'strand elements on that mask')
    # the reference decides Hs, the wave period and the wave direction over the whole element array; a shard sees only its own
    _distributed_refusal = 'ShipDrift'

    required_variables = {
        'x_wind': {'fallback': None},
        'y_wind': {'fallback': None},
        'land_binary_mask': {'fallback': None},
        'x_sea_water_velocity': {'fallback': None},
        'y_sea_water_velocity': {'fallback': None},
        'horizontal_diffusivity': {'fallback': 100, 'important': False},
        'sea_surface_wave_stokes_drift_x_velocity': {'fallback': 0},
        'sea_surface_wave_stokes_drift_y_velocity': {'fallback': 0},
        'sea_surface_wave_significant_height': {'fallback': 0},
        'sea_surface_wave_mean_period_from_variance_spectral_density_second_frequency_moment': {'fallback': 0}
    }

    winwav_angle = 20  # Angular offset in degrees

    def __init__(self, *args, wforce=None, **kwargs):
        path = wforce if wforce is not None else find_wforce()
        if path is None or not os.path.exists(path):
            raise FileNotFoundError('ShipDrift needs the wave force table wforce.dat: pass ShipDrift(wforce=<path to wforce.dat>) '
                                    '(no installed opendrift package provides models/wforce.dat)' if wforce is None else
                                    'ShipDrift(wforce=%r): no such file' % (wforce,))
        self.wforce = read_wforce(path)
        self.wforce_interpolator_F, self.wforce_interpolator_D = wforce_interpolators(self.wforce)
        self._wtab_host = wforce_table(self.wforce, self.wforce_interpolator_F)
        self._wtab_dev = None
        super().__init__(*args, **kwargs)
        self._add_config({'seed:orientation': {'type': 'enum', 'enum': ['left', 'right', 'random'], 'default': 'random',
                                               'level': CONFIG_LEVEL_ESSENTIAL,
                                               'description': 'If ships are oriented to the left or right of the downwind direction,'
                                                              'or whether this is unknown. Left/right means that wind will hit ship '
                                                              'from backboard/steerboard'},
                          'gpu:rng': {'type': 'enum', 'enum': ['numpy', 'philox'], 'default': 'numpy', 'level': CONFIG_LEVEL_ADVANCED,
                                      'description': 'numpy: the horizontal diffusion draws from the legacy generator on the host (bit '
                                                     'parity); philox: on the device, keyed by element ID.'}})
        self._set_config_default('drift:max_speed', 2)

    def seed_elements(self, *args, **kwargs):
        """shipdrift.py:157-214, including `len(kwargs[var] == 1)` (always true for a non-empty array)."""
        if 'number' in kwargs:
            num = kwargs['number']
        else:
            num = self.get_config('seed:number')
        for var in ['length', 'height', 'draft', 'beam']:
            if var not in kwargs:
                kwargs[var] = self.get_config('seed:' + var)
            kwargs[var] = np.atleast_1d(kwargs[var])
            if len(kwargs[var] == 1):
                kwargs[var] = kwargs[var] * np.ones(num)

        dl = kwargs['draft'] / kwargs['length']
        if dl.min() < 0.025 or dl.max() > 0.07:
            logger.warning('Ratio of draft to length should be in range 0.025 to 0.07, given range is %s-%s. Using border value.'
                           % (dl.min(), dl.max()))
            dl = np.clip(dl, 0.025, 0.07)
        bl = kwargs['beam'] / kwargs['length']
        if bl.min() < 0.12 or bl.max() > 0.18:
            logger.warning('Ratio of beam to length should be in range 0.12 to 0.18, given range is %s-%s. Using border value.'
                           % (bl.min(), bl.max()))

        # wind drag coefficient
        exposed = kwargs['height'] - kwargs['draft']
        Cf = np.zeros(num)
        Cf[exposed > 37.2] = 1.4
        Cf[exposed <= 37.2] = 1.045 + 0.016 * (exposed[exposed <= 37.2] - 15.)
        Cf[exposed <= 15] = 0.700 + 0.023 * exposed[exposed <= 15]
        kwargs['wind_drag_coeff'] = Cf

        # water drag coefficient
        beta = 2.0 * dl
        Cd = np.zeros(num)
        Cd[beta > .12] = 1.27
        Cd[beta <= .12] = 1.32 + (1.27 - 1.32) / 0.02 * (beta[beta <= .12] - 0.10)
        Cd[beta <= .10] = 1.38 + (1.32 - 1.38) / 0.02 * (beta[beta <= .10] - 0.08)
        Cd[beta <= .08] = 1.44 + (1.38 - 1.44) / 0.02 * (beta[beta <= .08] - 0.06)
        Cd[beta <= .06] = 1.50 + (1.44 - 1.50) / 0.01 * (beta[beta <= .06] - 0.05)
        kwargs['water_drag_coeff'] = Cd

        if 'orientation' not in kwargs:
            oc = self.get_config('seed:orientation')
            if oc == 'left':
                kwargs['orientation'] = np.ones(num) * 0
            elif oc == 'right':
                kwargs['orientation'] = np.ones(num) * 1
            else:
                kwargs['orientation'] = np.r_[:num] % 2  # Random 0 or 1

        super().seed_elements(*args, **kwargs)

    # -- physics_methods.py:893-943 on host arrays (for a subclass that runs its own update()) --------------------------------------
    def significant_wave_height(self):
        if HS in self.environment and self.environment.sea_surface_wave_significant_height.max() > 0:
            Hs = self.environment.sea_surface_wave_significant_height
        else:
            Hs = 0.0246 * np.power(self.wind_speed(), 2)
            setattr(self.environment, HS, np.asarray(Hs, dtype=np.float32))
        return Hs

    def _wave_frequency(self):
        windspeed = self.wind_speed()
        omega = 5 * np.ones(windspeed.shape)
        omega[windspeed > 0] = 0.877 * 9.81 / (1.17 * windspeed[windspeed > 0])
        return omega

    def wave_period(self):
        env = self.environment
        if TM02 in env and getattr(env, TM02).max() > 0:
            T = getattr(env, TM02).copy()
        elif TP in env and getattr(env, TP).max() > 0:
            T = getattr(env, TP).copy()
        else:
            T = (2 * np.pi) / self._wave_frequency()
            setattr(env, TM02, np.asarray(T, dtype=np.float32))
        if T.min() == 0:
            logger.warning('Zero wave period found - replacing with mean')
            T[T == 0] = np.mean(T[T > 0])
        return T

    # -- the device step ------------------------------------------------------------------------------------------------------------
    def _table(self):
        if self._wtab_dev is None:
            wtab, wbox, dims = self._wtab_host
            self._wtab_dev = (self.engine.to_device(wtab), self.engine.to_device(wbox), dims)
        return self._wtab_dev

    def _env_f32(self, name):
        """The step's float32 environment tensor of `name`, contiguous (kept in the environment)."""
        torch = self.engine.torch
        t = self.environment.dev(name, self.engine)
        if t.dtype != torch.float32 or not t.is_contiguous():
            t = t.to(torch.float32).contiguous()
            self.environment.set_dev(name, t)
        return t

    def _period_fill(self, T):
        """np.mean(T[T > 0]) of the float32 period in the reference's element order (NumPy's pairwise float32 sum depends on it):
        one copy of T to the host, made only on a step where some period is exactly 0."""
        torch = self.engine.torch
        if getattr(self, '_sorted', False):
            ids = self.elements.dev('ID').to(torch.int64)
            key = self.engine.to_device(self._release_rank)[ids - self._id_base]
            T = T[torch.argsort(key, stable=True)]
        Th = T.cpu().numpy()
        return np.mean(Th[Th > 0])

    def update(self):
        """shipdrift.py:216-343: the decisions over the whole array on the host, then one launch."""
        eng, el, torch = self.engine, self.elements, self.engine.torch
        n = len(el)
        if n == 0:
            return
        env = self.environment
        # wave_period(): Tm02, then Tp, then from the wind; zeros replaced by the mean
        T, tm_fill = None, None
        for name in (TM02, TP):
            if name in env:
                t = self._env_f32(name)
                lo, hi = eng.minmax(t)
                if hi > 0:
                    T = t
                    if lo == 0:
                        logger.warning('Zero wave period found - replacing with mean')
                        tm_fill = self._period_fill(t)
                    break
        tm_wind = T is None
        if tm_wind:
            T = torch.empty(n, dtype=torch.float32, device=eng.device)
            env.set_dev(TM02, T)
        # significant_wave_height(): the reader's, or from the wind
        hs_wind = not (HS in env and eng.minmax(self._env_f32(HS))[1] > 0)
        if hs_wind:
            hs = torch.empty(n, dtype=torch.float32, device=eng.device)
            env.set_dev(HS, hs)
        else:
            hs = self._env_f32(HS)
        # wave direction: the wind's when both Stokes maxima are 0
        sx, sy = self._env_f32(STOKES[0]), self._env_f32(STOKES[1])
        if eng.minmax(sx)[1] == 0 and eng.minmax(sy)[1] == 0:
            logger.info('Using wind direction as wave direction')
            sx = sy = None
        else:
            logger.info('Using Stokes drift direction as wave direction')
        cats = self.status_categories
        code = cats.index('ship stranded') if 'ship stranded' in cats else len(cats)
        envd = {'x_sea_water_velocity': self._env_f32('x_sea_water_velocity'), 'y_sea_water_velocity': self._env_f32('y_sea_water_velocity'),
                'x_wind': self._env_f32('x_wind'), 'y_wind': self._env_f32('y_wind'), 'hs': hs, 'period': T, 'stokes_x': sx,
                'stokes_y': sy, 'land_binary_mask': self._env_f32('land_binary_mask') if 'land_binary_mask' in env else None}
        eld = {k: el.dev(k, torch.float32) for k in SHIP_ELEMENTS}
        stranded = eng.ship_step(el.dev('lon', torch.float64), el.dev('lat', torch.float64), el.dev('moving', torch.int32),
                                 el.dev('status', torch.int32), eld, el.dev('orientation', torch.uint8), envd, self._table(),
                                 self.time_step.total_seconds(), hs_wind=hs_wind, tm_wind=tm_wind, tm_fill=tm_fill, strand_code=code)
        el.positions_f32 = False
        if stranded:
            if 'ship stranded' not in cats:
                cats.append('ship stranded')
            self._maybe_deactivated = True
