"""OpenDriftSimulation: the reference's run loop, seeding, configuration and element bookkeeping
(opendrift/models/basemodel/__init__.py) with particle state resident in HBM and the per-step arithmetic in
libodcuda.so.

Same public surface as the reference for the advection path:
  __init__(seed=0, loglevel=...), add_reader(), set_config()/get_config(), seed_elements(), run(time_step, steps,
  duration, end_time, time_step_output), update() (abstract), update_positions(x_vel, y_vel),
  horizontal_diffusion(), deactivate_elements(), elements / elements_deactivated / environment / time / time_step,
  num_elements_active()/..., get_lonlats().
Not rebuilt (out of scope, SURVEY.md section 2): plotting/animation, netCDF/parquet export, landmask/coastline
interaction, seafloor interaction, lazy readers, the xarray result Dataset (a NumPy history buffer stands in).

Reference line numbers are cited at each method.
"""
import logging
from datetime import timedelta

import numpy as np

from ..config import Configurable, CONFIG_LEVEL_ESSENTIAL, CONFIG_LEVEL_BASIC, CONFIG_LEVEL_ADVANCED
from ..elements import LagrangianArray, DeviceElements
from ..engine import default_engine
from .environment import Environment
from .physics_methods import PhysicsMethods

logger = logging.getLogger('opendrift_b200')


class EnvironmentView:
    """self.environment: attribute access returns float32 NumPy arrays like the reference's recarray;
    the data are device tensors sampled at the start of the step."""

    def __init__(self, tensors):
        object.__setattr__(self, '_t', tensors)
        object.__setattr__(self, '_h', {})

    def __getattr__(self, name):
        t = object.__getattribute__(self, '_t')
        h = object.__getattribute__(self, '_h')
        if name in h:
            return h[name]
        if name in t:
            h[name] = t[name].cpu().numpy()
            t.pop(name)                # host copy is now authoritative (may be modified in place)
            return h[name]
        raise AttributeError(name)

    def __setattr__(self, name, value):
        self._h[name] = np.asarray(value)
        self._t.pop(name, None)

    def dev(self, name, engine):
        if name in self._h:
            self._t[name] = engine.to_device(np.ascontiguousarray(self._h.pop(name)))
        return self._t[name]

    def __contains__(self, name):
        return name in self._t or name in self._h

    def permute(self, perm, engine):
        """Re-order the rows as the element arrays were re-ordered (row k <- row perm[k])."""
        t, h = object.__getattribute__(self, '_t'), object.__getattribute__(self, '_h')
        for k in list(t):
            t[k] = engine.permute(perm, t[k]) if t[k].dim() == 1 else t[k][perm.long()]
        if h:
            ph = perm.cpu().numpy()
            for k in list(h):
                h[k] = h[k][ph]

    def select(self, keep):
        """Keep the rows of the elements selected by the boolean device tensor `keep`."""
        t, h = object.__getattribute__(self, '_t'), object.__getattribute__(self, '_h')
        for k in list(t):
            t[k] = t[k][keep]
        if h:
            kh = keep.cpu().numpy()
            for k in list(h):
                h[k] = h[k][kh]


class ResultVariable:
    """result.<var>: `.values` is the [trajectory, time] array of the reference's xr.DataArray."""

    def __init__(self, rows, name):
        self._rows, self.name = rows, name

    @property
    def values(self):
        if self.name == 'time':
            return np.array(self._rows)
        return np.array(self._rows).T if len(self._rows) else np.zeros((0, 0), dtype=np.float32)

    def __array__(self, dtype=None, copy=None):
        v = self.values
        return v if dtype is None else v.astype(dtype)

    def isel(self, time=None, trajectory=None):
        v = self.values
        if self.name == 'time':
            return v if time is None else v[time]
        if trajectory is not None:
            v = v[trajectory]
        if time is not None:
            v = v[..., time]
        return v

    def min(self):
        return np.nanmin(self.values)

    def max(self):
        return np.nanmax(self.values)


class Result(dict):
    """What run() returns and o.result holds.  The reference returns an xr.Dataset with lon / lat / z / status [trajectory, time]
    (basemodel/__init__.py:2100-2135, 2340); xarray is outside this package's dependencies, so the same data come as a dict of
    per-output-time rows -- result['lon'][k] is the float32 [trajectory] array of output time result['time'][k], NaN (status -1)
    where the element does not exist -- with the Dataset's access pattern on top: result.lon.values is [trajectory, time],
    result.time.values the time axis, result.sizes, result.status_categories (the flag_meanings of the status variable)."""

    status_categories = ()

    def __getattr__(self, name):
        if name in self:
            return ResultVariable(self[name], name)
        raise AttributeError(name)

    @property
    def sizes(self):
        return {'time': len(self['time']), 'trajectory': len(self['lon'][0]) if self['lon'] else 0}

    @property
    def data_vars(self):
        return [k for k in self if k != 'time']


class OpenDriftSimulation(PhysicsMethods, Configurable):
    ElementType = LagrangianArray
    required_variables = {}
    status_categories = ['active']

    def __init__(self, seed=0, loglevel=None, logfile=None, engine=None, **kwargs):
        Configurable.__init__(self)
        self.status_categories = ['active']
        if seed is not None:
            np.random.seed(seed)                      # basemodel/__init__.py:326: the legacy global generator
        self._seed = 0 if seed is None else int(seed)
        self._engine = engine
        self.origin_marker = None
        self.steps_calculation = 0
        self.elements_deactivated = self.ElementType()
        self.env = Environment(self.required_variables, self)
        self.validity_domain = None
        self.history = None
        c = {
            'general:time_step_minutes': {'type': 'float', 'min': .01, 'max': 1440, 'default': 60, 'units': 'minutes',
                                          'level': CONFIG_LEVEL_BASIC, 'description': 'Calculation time step.'},
            'general:time_step_output_minutes': {'type': 'float', 'min': 1, 'max': 1440, 'default': None,
                                                 'units': 'minutes', 'level': CONFIG_LEVEL_BASIC,
                                                 'description': 'Output time step.'},
            'general:use_auto_landmask': {'type': 'bool', 'default': True, 'level': CONFIG_LEVEL_ADVANCED,
                                          'description': 'Accepted for script compatibility; no landmask on the GPU path.'},
            'general:coastline_action': {'type': 'enum', 'enum': ['none', 'stranding', 'previous'], 'default': 'none',
                                         'level': CONFIG_LEVEL_BASIC,
                                         'description': 'None, or stranding / previous against the land_binary_mask of a gridded reader '
                                                        '(with general:coastline_approximation_precision = None).'},
            'seed:number': {'type': 'int', 'default': 1, 'min': 1, 'max': 100000000, 'units': 1,
                            'level': CONFIG_LEVEL_BASIC, 'description': 'The number of elements for the simulation.'},
            # keys the reference's scripts set that concern subsystems outside the GPU path: accepted with the reference's
            # defaults so that set_config does not raise; values that would change the physics are refused at run()
            'general:simulation_name': {'type': 'str', 'min_length': 0, 'max_length': 64, 'default': '', 'level': CONFIG_LEVEL_BASIC,
                                        'description': 'Name of simulation'},
            'general:coastline_approximation_precision': {'type': 'float', 'default': 0.001, 'min': 0.0001, 'max': 0.005, 'units': 'degrees',
                                                          'level': CONFIG_LEVEL_ADVANCED,
                                                          'description': 'The bisection towards the GSHHG coastline is IO-backed (roaring_landmask) and not on the GPU path: '
                                                                         'set to None when general:coastline_action is not none.'},
            'general:seafloor_action': {'type': 'enum', 'enum': ['none', 'lift_to_seafloor', 'deactivate', 'previous'],
                                        'default': 'lift_to_seafloor', 'level': CONFIG_LEVEL_ADVANCED,
                                        'description': 'Accepted for script compatibility: seafloor interaction needs a bathymetry reader '
                                                       '(outside the GPU path); with the 10 km fallback depth no element ever reaches it.'},
            'readers:max_number_of_fails': {'type': 'int', 'default': 1, 'min': 0, 'max': 1e6, 'units': 'number', 'level': CONFIG_LEVEL_ADVANCED,
                                            'description': 'Accepted for script compatibility (in-memory readers do not fail).'},
            'drift:profiles_depth': {'type': 'float', 'default': 50, 'min': 0, 'max': None, 'units': 'meters', 'level': CONFIG_LEVEL_ADVANCED,
                                     'description': 'Accepted for script compatibility: the mixing kernel reads the whole column of the block.'},
            'seed:ocean_only': {'type': 'bool', 'default': True, 'level': CONFIG_LEVEL_ESSENTIAL,
                                'description': 'Accepted for script compatibility: moving elements seeded on land to the closest '
                                               'ocean point needs a landmask, which is outside the GPU path.'},
            'seed:seafloor': {'type': 'bool', 'default': False, 'level': CONFIG_LEVEL_ESSENTIAL,
                              'description': 'Elements are seeded at seafloor (needs a bathymetry reader: not on the GPU path).'},
            'drift:max_age_seconds': {'type': 'float', 'default': None, 'min': 0, 'max': np.inf, 'units': 'seconds',
                                      'level': CONFIG_LEVEL_ADVANCED, 'description': 'Retire elements at this age.'},
            'drift:advection_scheme': {'type': 'enum', 'enum': ['euler', 'runge-kutta', 'runge-kutta4'],
                                       'default': 'euler', 'level': CONFIG_LEVEL_ADVANCED,
                                       'description': 'Numerical advection scheme for ocean current advection'},
            'drift:max_speed': {'type': 'float', 'default': 1, 'min': 0, 'max': np.inf, 'units': 'm/s',
                                'level': CONFIG_LEVEL_ESSENTIAL, 'description': 'Maximum anticipated speed.'},
            'drift:current_uncertainty': {'type': 'float', 'default': 0, 'min': 0, 'max': 5, 'units': 'm/s',
                                          'level': CONFIG_LEVEL_ADVANCED,
                                          'description': 'Add gaussian perturbation with this standard deviation to current components at each time step'},
            'drift:current_uncertainty_uniform': {'type': 'float', 'default': 0, 'min': 0, 'max': 5, 'units': 'm/s',
                                                  'level': CONFIG_LEVEL_ADVANCED,
                                                  'description': 'Add gaussian perturbation with this magnitude to current components at each time step'},
            'drift:wind_uncertainty': {'type': 'float', 'default': 0, 'min': 0, 'max': 5, 'units': 'm/s',
                                       'level': CONFIG_LEVEL_ADVANCED,
                                       'description': 'Add gaussian perturbation with this standard deviation to wind components at each time step.'},
            'drift:relative_wind': {'type': 'bool', 'default': False, 'level': CONFIG_LEVEL_ADVANCED,
                                    'description': 'Wind relative to the ocean current.'},
            'drift:deactivate_north_of': {'type': 'float', 'default': None, 'min': -90, 'max': 90, 'units': 'degrees',
                                          'level': CONFIG_LEVEL_ADVANCED, 'description': 'Deactivate north of.'},
            'drift:deactivate_south_of': {'type': 'float', 'default': None, 'min': -90, 'max': 90, 'units': 'degrees',
                                          'level': CONFIG_LEVEL_ADVANCED, 'description': 'Deactivate south of.'},
            'drift:deactivate_east_of': {'type': 'float', 'default': None, 'min': -360, 'max': 360, 'units': 'degrees',
                                         'level': CONFIG_LEVEL_ADVANCED, 'description': 'Deactivate east of.'},
            'drift:deactivate_west_of': {'type': 'float', 'default': None, 'min': -360, 'max': 360, 'units': 'degrees',
                                         'level': CONFIG_LEVEL_ADVANCED, 'description': 'Deactivate west of.'},
            'gpu:sort_interval_steps': {'type': 'int', 'default': 20, 'min': 0, 'max': 1000000, 'units': 1,
                                        'level': CONFIG_LEVEL_ADVANCED,
                                        'description': 'Re-order the device particle arrays by grid cell every N steps (0 = never).'},
            'gpu:history': {'type': 'enum', 'enum': ['host', 'device'], 'default': 'device', 'level': CONFIG_LEVEL_ADVANCED,
                            'description': 'Where the output buffer of state_to_buffer lives between flushes: device = a block of output '
                                           'columns in HBM, filled by the per-step bookkeeping launch and read back once per '
                                           'export_buffer_length output steps; host = a block of one column (read back every output step).'},
            'gpu:history_pinned_bytes': {'type': 'int', 'default': 16 * 2 ** 30, 'min': 0, 'max': 2 ** 44, 'units': 'bytes',
                                         'level': CONFIG_LEVEL_ADVANCED,
                                         'description': 'Outputs with more columns than one device block: the host side of the output buffer is '
                                                        'page-locked memory (full blocks then travel asynchronously on the copy stream) when the '
                                                        'whole time axis fits this many bytes; 0 = always pageable.'},
            'gpu:distributed': {'type': 'bool', 'default': True, 'level': CONFIG_LEVEL_ADVANCED,
                                'description': 'Under torchrun (torch.distributed initialised, one process per GPU): rank 0 reads the forcing '
                                               'slabs and broadcasts them into the other ranks\' device ring; ranks step in lockstep.'},
            'gpu:shard': {'type': 'enum', 'enum': ['index', 'none'], 'default': 'index', 'level': CONFIG_LEVEL_ADVANCED,
                          'description': 'Distributed runs: index = every rank seeded all elements (same script) and keeps a contiguous '
                                         'index range of them; none = the script seeded only this rank\'s elements.'},
            'gpu:history_block_bytes': {'type': 'int', 'default': 2 ** 31, 'min': 1, 'max': 2 ** 40, 'units': 'bytes',
                                        'level': CONFIG_LEVEL_ADVANCED,
                                        'description': 'Upper bound of the device block of output columns (16 bytes per element and column).'},
            'gpu:arithmetic': {'type': 'enum', 'enum': ['series', 'exact', 'fast'], 'default': 'series', 'level': CONFIG_LEVEL_ADVANCED,
                               'description': 'Arithmetic of the step kernels (include/odcuda.h OD_MATH_*): series = bit-exact field '
                                              'sampling + short-arc series geodesic (round-off accurate); exact = the reference\'s '
                                              'arithmetic operation by operation (full Karney geodesic, float32 mid-point azimuths); '
                                              'fast = float32 sampling (within ~3e-8 deg of the reference on the fixtures).'},
        }
        # environment:constant:<var> / environment:fallback:<var> per required variable (environment.py:41-76)
        for v, spec in self.required_variables.items():
            c['environment:constant:%s' % v] = {'type': 'float', 'min': None, 'max': None, 'units': '', 'default': None,
                                                'level': CONFIG_LEVEL_BASIC, 'description': 'Constant value for %s' % v}
            c['environment:fallback:%s' % v] = {'type': 'float', 'min': None, 'max': None, 'units': '',
                                                'default': spec.get('fallback'), 'level': CONFIG_LEVEL_BASIC,
                                                'description': 'Fallback value for %s' % v}
        self._add_config(c)
        # seed:<property> for element properties with a default (used by seed_elements)
        for name, spec in self.ElementType.variables.items():
            if spec.get('seed', True) and 'default' in spec:
                self._add_config({'seed:%s' % name: {'type': 'float', 'min': None, 'max': None, 'units': '',
                                                      'default': spec['default'], 'level': CONFIG_LEVEL_BASIC,
                                                      'description': 'Seed property %s' % name}}, overwrite=False)

    # ------------------------------------------------------------------------------------------------
    @property
    def engine(self):
        if self._engine is None:
            self._engine = default_engine()
        return self._engine

    def add_reader(self, readers, variables=None, first=False):
        self.env.add_reader(readers, variables, first)

    def add_readers_from_list(self, *a, **k):
        raise NotImplementedError('lazy readers are host-side IO, out of scope of the GPU hot path')

    # -- counts (basemodel/__init__.py:841-866) ----------------------------------------------------------
    def num_elements_active(self):
        return len(self.elements) if hasattr(self, 'elements') else 0

    def num_elements_scheduled(self):
        return len(self.elements_scheduled) if hasattr(self, 'elements_scheduled') else 0

    def num_elements_deactivated(self):
        return len(self.elements_deactivated)

    def num_elements_activated(self):
        return self.num_elements_active() + self.num_elements_deactivated()

    def num_elements_total(self):
        return self.num_elements_activated() + self.num_elements_scheduled()

    # -- seeding (basemodel/__init__.py:1033-1237, 869-907) ------------------------------------------------
    def seed_elements(self, lon, lat, time, radius=0, number=None, number_per_point=None,
                      radius_type='gaussian', **kwargs):
        if self.origin_marker is None:
            self.origin_marker = {}
        kwargs.setdefault('origin_marker', len(self.origin_marker))
        self.origin_marker[str(kwargs['origin_marker'])] = kwargs.pop('origin_marker_name',
                                                                      'Seed %d' % len(self.origin_marker)).replace(' ', '_')
        lon = np.atleast_1d(lon).ravel()
        lat = np.atleast_1d(lat).ravel()
        radius = np.atleast_1d(radius).ravel()
        time = list(np.atleast_1d(time))
        if lat.max() > 90 or lat.min() < -90:
            raise ValueError('Latitude must be between -90 and 90 degrees')
        if len(lon) != len(lat):
            raise ValueError('Lon and lat must have same lengths')
        if len(lon) > 1:
            if number_per_point is not None:
                if number is not None:
                    raise ValueError('Both number and number_per_point is provided')
                number = number_per_point * len(lon)
            if number is not None:
                if number % len(lon) != 0:
                    raise ValueError('Lon and lat have length %s, but number is %s, which is not a multiple'
                                     % (len(lon), number))
                npp = int(number / len(lon))
                if npp > 1:
                    lon, lat = np.repeat(lon, npp), np.repeat(lat, npp)
            number = len(lon)
        else:
            if number is None:
                number = len(time) if len(time) > 2 else self.get_config('seed:number')
            lon = lon * np.ones(number)
            lat = lat * np.ones(number)
        if len(time) != number and len(time) > 1:
            if len(time) == 2:
                td = (time[1] - time[0]) / (number - 1)
                time = [time[0] + i * td for i in range(number)]
            else:
                raise ValueError('Time array has length %s, must be 1, 2 or %s' % (len(time), number))
        if radius.max() > 0:
            # same draws, same order as the reference (:1150-1166); the geodesic runs on the GPU
            if radius_type == 'gaussian':
                x = np.random.randn(number) * radius
                y = np.random.randn(number) * radius
                az = np.degrees(np.arctan2(x, y))
                dist = np.sqrt(x * x + y * y)
            elif radius_type == 'uniform':
                az = np.random.rand(number) * 360
                dist = np.sqrt(np.random.uniform(0, 1, number)) * radius
            else:
                raise ValueError('unknown radius_type ' + str(radius_type))
            eng = self.engine
            d_lon, d_lat = eng.to_device(lon.astype(np.float64)), eng.to_device(lat.astype(np.float64))
            eng.geod_fwd(d_lon, d_lat, eng.to_device(az.astype(np.float64)), eng.to_device(dist.astype(np.float64)))
            lon, lat = d_lon.cpu().numpy(), d_lat.cpu().numpy()
        if isinstance(kwargs.get('z'), str) or (kwargs.get('z') is None and self.get_config('seed:seafloor', False)):
            raise NotImplementedError("z='seafloor' / seed:seafloor needs a bathymetry reader, which is outside the GPU path")
        for key, spec in self.get_configspec('seed:').items():
            prop = key.split(':')[-1]
            if prop not in kwargs and prop in self.ElementType.variables:
                kwargs[prop] = spec['value']
        elements = self.ElementType(lon=lon, lat=lat, **kwargs)
        return self.schedule_elements(elements, time)

    def schedule_elements(self, elements, time):
        if len(time) == 1 and len(elements) > 1:
            time = time * len(elements)
        if not hasattr(self, 'elements_scheduled'):
            self.elements_scheduled = elements
            self.elements_scheduled_time = np.array(time)
            self.start_time = time[0]
            self.elements_scheduled.ID = np.arange(0, len(elements))
        else:
            elements.ID = np.arange(self.num_elements_scheduled(), self.num_elements_scheduled() + len(elements))
            self.elements_scheduled.extend(elements)
            self.elements_scheduled_time = np.append(self.elements_scheduled_time, np.array(time))
        self.start_time = min(self.start_time, min(time))
        return elements.ID

    def release_elements(self):
        """:909-934 -- scheduled elements whose time falls inside this step move to the device arrays."""
        if len(self.elements_scheduled) == 0:
            self._newly_seeded = False                         # newly_seeded_IDs = None (:916-918)
            return
        self._newly_seeded = True                              # (an array, possibly empty: 'is not None' in interact_with_coastline)
        t, dt = self.time, self.time_step
        st = self.elements_scheduled_time
        idx = (st >= t) & (st < t + dt) if dt.days >= 0 else (st <= t) & (st > t + dt)
        if not idx.any():
            return
        first_release = len(self.elements) == 0
        ids = np.asarray(self.elements_scheduled.ID)[idx].astype(np.int64)
        if getattr(self, '_store_previous', False):
            # _elements_previous.lon[newly_seeded_IDs] = elements_scheduled.lon[indices] (:928-931): float32 like the result block
            k = self.engine.to_device(ids - self._id_base)
            self._prev_lon[k] = self.engine.to_device(np.asarray(self.elements_scheduled.lon)[idx].astype(np.float32))
            self._prev_lat[k] = self.engine.to_device(np.asarray(self.elements_scheduled.lat)[idx].astype(np.float32))
        self._release_rank[ids - self._id_base] = np.arange(self._released, self._released + len(ids))     # the reference's array order
        self._released += len(ids)
        self.elements.append_host(self.elements_scheduled, idx)
        keep = self.ElementType()
        self.elements_scheduled.move_elements(keep, idx)      # drops the released ones from the schedule
        self.elements_scheduled_time = st[~idx]
        if not first_release:
            self.elements.positions_f32 = False                # mixed ages: already float64 positions

    # -- deactivation (:1774-1826) ---------------------------------------------------------------------------
    def deactivate_elements(self, indices, reason='deactivated'):
        torch = self.engine.torch
        if isinstance(indices, np.ndarray):
            if not indices.any():
                return
            indices = self.engine.to_device(indices.astype(bool))
        elif not bool(indices.any()):
            return
        if reason not in self.status_categories:
            self.status_categories.append(reason)
        code = self.status_categories.index(reason)
        status = self.elements.dev('status')
        moving = self.elements.dev('moving')
        self.elements.set_dev('status', torch.where(indices & (status == 0), torch.full_like(status, code), status))
        self.elements.set_dev('moving', torch.where(indices, torch.zeros_like(moving), moving))
        self._maybe_deactivated = True

    def remove_deactivated_elements(self):
        if not getattr(self, '_maybe_deactivated', False) or len(self.elements) == 0:
            return
        self._maybe_deactivated = False
        pre = getattr(self, '_noise0', None)
        view = getattr(self, '_env_view', None)
        keep = keep_dev = None
        ssh = getattr(self, '_ssh_now', None)
        if pre or view is not None or ssh is not None:
            keep_dev = self.elements.dev('status') == 0
            if pre:
                keep = keep_dev.cpu().numpy()
        removed = self.elements.compact()
        if pre and removed is not None:
            for k in pre:
                pre[k] = [a[keep] for a in pre[k]]
        if view is not None and removed is not None:       # self.environment = self.environment[~indices] (:1812-1813)
            view.select(keep_dev)
        if ssh is not None and removed is not None:
            self._ssh_now = ssh[keep_dev]
        if removed is None:
            return
        tmp = self.ElementType(**{k: v for k, v in removed.items()})
        for k, v in removed.items():                           # keep the dtypes the active arrays had
            setattr(tmp, k, v)
        sel = np.ones(len(tmp), dtype=bool)
        tmp.move_elements(self.elements_deactivated, sel)
        self._env_dev = None

    # -- per-step housekeeping: one launch (od_bookkeeping) ------------------------------------------------------
    def _bookkeep(self, outside=True, buffer_col=None, only_deactivated=False, age=True):
        """deactivate_outside (:2358-2386) -> state_to_buffer (:2384-2403) -> increase_age_and_retire (:2345-2356) for the
        active elements, in the reference's order, as ONE kernel launch.  The host is only synchronised (a 12-byte read of the
        kernel's counters) when something CAN have been deactivated: a validity domain or a maximum age is configured, or an
        earlier launch / a subclass flagged elements; the compaction is skipped when nothing was."""
        n = self.num_elements_active()
        if n == 0:
            return
        eng, el, torch = self.engine, self.elements, self.engine.torch
        cats = self.status_categories
        domain = self.validity_domain if outside else None
        max_age = self.get_config('drift:max_age_seconds') if age else None
        new_out = domain is not None and 'outside' not in cats
        oc = cats.index('outside') if 'outside' in cats else len(cats)
        rc = cats.index('retired') if 'retired' in cats else len(cats) + (1 if new_out else 0)
        if getattr(el, 'status_touched', False):          # a subclass assigned / was handed elements.status (host view)
            self._maybe_deactivated = True
            el.status_touched = False
        counts = domain is not None or max_age is not None or self._maybe_deactivated
        agev = el.dev('age_seconds')
        if agev.dtype not in (torch.float32, torch.float64):
            agev = el.dev('age_seconds', torch.float64)
        buf = None
        if buffer_col is not None:
            buf = self._hist_column(buffer_col)
        res = eng.bookkeeping(el.dev('lon', torch.float64), el.dev('lat', torch.float64), self._z_for_sampling(), agev,
                              el.dev('status', torch.int32), el.dev('moving', torch.int32), el.dev('ID', torch.int32),
                              self.time_step.total_seconds() if age else 0.0, max_age, domain, oc, rc,
                              pos_f32=el.positions_f32, buf=buf, only_deactivated=only_deactivated, counts=counts,
                              id_base=self._id_base)
        if res is None:
            return
        n_out, n_ret, n_off = res
        if new_out and n_out > 0:                          # a category is numbered when it first occurs (:1778-1780)
            cats.append('outside')
        if n_ret > 0 and 'retired' not in cats:
            cats.append('retired')
            real = cats.index('retired')
            if real != rc:                                 # 'outside' was provisionally numbered before it and did not occur
                st = el.dev('status')
                el.set_dev('status', torch.where(st == rc, torch.full_like(st, real), st))
        self._maybe_deactivated = n_off > 0

    def increase_age_and_retire(self):
        """:2345-2356"""
        self._bookkeep(outside=False, age=True)

    def deactivate_outside(self):
        """:2358-2386"""
        if self.validity_domain is not None:
            self._bookkeep(outside=True, age=False)

    def _setup_coastline(self):
        """general:coastline_action against a land_binary_mask that a gridded reader provides.  The reference's default -- the GSHHG
        landmask of roaring_landmask, loaded when general:use_auto_landmask is on, and the bisection of coastline_crossing
        against it -- is IO-backed and not on this path."""
        self._coast = None
        self._store_previous = False
        if self.get_config('general:seafloor_action') == 'previous' and self.env.priority_list.get('sea_floor_depth_below_sea_level'):
            self._alloc_previous()
        action = self.get_config('general:coastline_action')
        if action == 'none' and self.env.priority_list.get('land_binary_mask') \
                and self._config['general:coastline_action'].get('value') == self._config['general:coastline_action'].get('default') \
                and not getattr(self, '_coast_default_warned', False):
            # The reference's default is 'stranding' (against the GSHHG landmask, which is not on this path); the default here is
            # 'none'.  A script that adds a land_binary_mask reader and leaves the action alone would strand under the reference.
            self._coast_default_warned = True
            logger.warning("a reader provides land_binary_mask but general:coastline_action is 'none' (the default of the GPU classes; the "
                           "reference's default is 'stranding'): set general:coastline_action = 'stranding' and "
                           "general:coastline_approximation_precision = None to strand elements on that mask")
        if action == 'none' or 'land_binary_mask' not in self.required_variables:
            return
        if self.env.constant('land_binary_mask') is not None and not self.env.priority_list.get('land_binary_mask'):
            if float(self.env.constant('land_binary_mask')) == 0:
                return                                        # no land anywhere
            raise NotImplementedError('environment:constant:land_binary_mask = 1 (land everywhere) is not a case for the GPU path')
        if not self.env.priority_list.get('land_binary_mask'):
            raise NotImplementedError("general:coastline_action = '%s' needs a reader that provides land_binary_mask; the GSHHG landmask "
                                      "(general:use_auto_landmask) is host-side IO, out of scope of the GPU hot path" % action)
        if self.get_config('seed:ocean_only'):
            # "Move point seeded on land to ocean" (:2148-2155), once, before the run, on the scheduled (float32) positions
            lon, lat = np.asarray(self.elements_scheduled.lon), np.asarray(self.elements_scheduled.lat)
            lon, lat, _ = self.closest_ocean_points(lon, lat)
            self.elements_scheduled.lon, self.elements_scheduled.lat = lon, lat
        if self.get_config('general:coastline_approximation_precision') is not None:
            raise NotImplementedError('general:coastline_approximation_precision must be None on the GPU path: the bisection towards '
                                      'the coastline queries the GSHHG landmask (basemodel/__init__.py:81-134)')
        if action == 'previous' and not getattr(self, '_coast_previous_supported', False):
            # an element that is moved back keeps, for this step, the environment sampled where it was on land (the reference samples
            # before interact_with_coastline, :2238-2253): only models whose update() can run from a materialised environment do that
            raise NotImplementedError("general:coastline_action = 'previous' is not on the GPU path of %s" % type(self).__name__)
        self._coast = action
        self._alloc_previous()

    def closest_ocean_points(self, lon, lat):
        """:936-1030 for a gridded land_binary_mask reader: the seeds on land (mask != 0, which includes 'no data') move to the
        nearest ocean point of a 0.01 degree grid around the seeds (<= 1000 points per axis), as sampled from the same reader at its
        start time; a k-d tree search on the host, once per run (scipy, like the reference).  Positions keep their dtype."""
        from scipy.spatial import cKDTree
        name = self.env.priority_list['land_binary_mask'][0]
        land_reader = self.env.readers[name]
        lon, lat = np.array(lon, copy=True), np.array(lat, copy=True)
        deltalon = deltalat = 0.01
        numbuffer = 10
        lonmin, lonmax = lon.min() - deltalon * numbuffer, lon.max() + deltalon * numbuffer
        latmin, latmax = lat.min() - deltalat * numbuffer, lat.max() + deltalat * numbuffer
        sample = lambda x, y: self.env.get_environment(['land_binary_mask'], lon=x, lat=y, z=0 * x,            # noqa: E731
                                                       time=land_reader.start_time)[0]['land_binary_mask']
        land = sample(lon, lat)
        if land.max() == 0:
            return lon, lat, None
        land_indices = np.where(land != 0)[0]
        longrid = np.arange(lonmin, lonmax, deltalon)
        latgrid = np.arange(latmin, latmax, deltalat)
        if len(longrid) > 1000 or len(latgrid) > 1000:
            longrid = np.linspace(lonmin, lonmax, 1000)
            latgrid = np.linspace(latmin, latmax, 1000)
        longrid, latgrid = np.meshgrid(longrid, latgrid)
        longrid, latgrid = longrid.ravel(), latgrid.ravel()
        covered = land_reader.covers_positions(longrid, latgrid)[0]
        longrid, latgrid = longrid[covered], latgrid[covered]
        if longrid.size == 0:
            return lon, lat, land_indices
        landgrid = sample(longrid, latgrid)
        if landgrid.size == 0 or landgrid.min() == 1 or np.isnan(landgrid.min()):
            return lon, lat, land_indices                      # 'No ocean pixels nearby, cannot move elements.'
        olon, olat = longrid[landgrid == 0], latgrid[landgrid == 0]
        tree = cKDTree(np.dstack([olon, olat])[0])
        _dist, idx = tree.query(np.dstack([lon[land_indices], lat[land_indices]]))
        idx = idx.ravel()
        lon[land_indices] = olon[idx]
        lat[land_indices] = olat[idx]
        return lon, lat, land_indices

    def _alloc_previous(self):
        """lon / lat of the previous step, float32, one row per trajectory: the reference's `_elements_previous` (a copy of its
        float32 result block, :2164-2165; kept when a coastline or sea-floor action may move elements back, elements.py:76-88)."""
        if self._store_previous:
            return
        torch = self.engine.torch
        n = len(self._release_rank)
        self._store_previous = True
        self._prev_lon = torch.full((n,), float('nan'), dtype=torch.float32, device=self.engine.device)
        self._prev_lat = torch.full((n,), float('nan'), dtype=torch.float32, device=self.engine.device)

    def interact_with_coastline(self, final=False):
        """:671-746 -- 'stranding': elements on land (and not in the air) are deactivated; 'previous': elements released on land are
        deactivated ('seeded_on_land'), every element on land goes back to its position of the previous step.  One sampling launch
        (nearest grid point of the mask) and one launch for the action; elements the mask reader does not cover become
        'missing_data' (report_missing_variables, :2501-2515; not at the final call)."""
        if getattr(self, '_coast', None) is None or self.num_elements_active() == 0:
            return
        eng, el, torch = self.engine, self.elements, self.engine.torch
        cats = self.status_categories
        mask = self._start_of_step_sample('land_binary_mask')
        if self._vertical_advection_correction():
            # an element with an undefined depth is not covered by the mask reader (see report_missing_variables): NaN, no action
            mask = torch.where(torch.isnan(self._z_for_sampling()), torch.full_like(mask, float('nan')), mask)
        self._coast_moved = False
        if self._coast == 'previous' and not final and bool((mask == 1).any()):
            # Elements on land go back to where they were, but update() still sees the environment sampled where they are now
            # (the reference samples the step's environment before this method, :2238-2253, and does not sample again): materialise
            # it before the move; this step then runs from it (the fused step would sample at the restored positions).
            _ = self.environment
            self._coast_moved = True
        names = ['missing_data'] + (['stranded'] if self._coast == 'stranding' else ['seeded_on_land'])
        prov, nxt = {}, len(cats)
        for nm in names:
            if nm in cats:
                prov[nm] = cats.index(nm)
            else:
                prov[nm], nxt = nxt, nxt + 1
        age = el.dev('age_seconds')
        if age.dtype not in (torch.float32, torch.float64):
            age = age.to(torch.float64)
        lon, lat = el.dev('lon', torch.float64), el.dev('lat', torch.float64)
        n_str, n_seed, n_miss, n_back = eng.coastline(
            mask, lon, lat, self._z_for_sampling(), age, el.dev('status', torch.int32), el.dev('moving', torch.int32),
            el.dev('ID', torch.int32), self._prev_lon, self._prev_lat, self._id_base, self._coast,
            stranded_code=prov.get('stranded', 0), seeded_code=prov.get('seeded_on_land', 0),
            missing_code=0 if final else prov['missing_data'], check_seeded=getattr(self, '_newly_seeded', False))
        el.set_dev('lon', lon)
        el.set_dev('lat', lat)
        # categories are numbered when they first occur, missing_data (reported at the top of the loop) before the coastline's
        for nm, cnt in (('missing_data', n_miss), (names[1], n_str + n_seed)):
            if cnt > 0 and nm not in cats:
                cats.append(nm)
                real = cats.index(nm)
                if real != prov[nm]:
                    st = el.dev('status')
                    el.set_dev('status', torch.where(st == prov[nm], torch.full_like(st, real), st))
        if n_str + n_seed + n_miss > 0:
            self._maybe_deactivated = True

    def _variables_that_may_miss(self):
        """Variables a reader provides and for which neither a constant nor a fallback value is configured
        (`environment:fallback:<variable>` = None): outside the readers' coverage they are missing."""
        return [v for v in getattr(self, '_env_variables', ())
                if self.env.priority_list.get(v) and self.env.constant(v) is None and self.env.fallback(v) is None
                and not (v == 'land_binary_mask' and getattr(self, '_coast', None) is not None)]    # (interact_with_coastline reports it)

    def report_missing_variables(self):
        """:2249, 2501-2515 -- elements for which a variable without fallback value is missing (outside the readers' coverage, no data
        there, or a position that an earlier Runge-Kutta stage without forcing has left undefined) leave as 'missing_data' at the
        top of the loop.  Costs nothing with the default configuration (every variable of the stock recipes has a fallback value);
        otherwise those variables are sampled here, before deactivate_outside as in the reference."""
        may_miss = self._variables_that_may_miss()
        # No reader covers an element with an undefined depth: the reference's coverage test is zmin <= z <= zmax for gridded, 2-D
        # and constant readers alike (readers/basereader/variables.py:241-251), so a variable without a fallback value is missing
        # there, wherever it comes from (the device samplers of 2-D fields do not look at z).  Undefined depths come from
        # drift:vertical_advection_correction: an element without a previous sea surface height (update_previous_state)
        nan_z = self._vertical_advection_correction() and any(self.env.fallback(v) is None for v in getattr(self, '_env_variables', ()))
        if (not may_miss and not nan_z) or self.num_elements_active() == 0:
            return
        el, torch = self.elements, self.engine.torch
        missing = None
        if may_miss:
            _, missing = self.env.device_environment(may_miss, self.time, el.dev('lon', torch.float64), el.dev('lat', torch.float64),
                                                     self._z_truncated(), pos_f32=el.positions_f32)
        if nan_z:
            undefined = torch.isnan(self._z_for_sampling())
            missing = undefined if missing is None else (missing | undefined)
        self._deactivate_missing(missing)

    def _deactivate_missing(self, missing):
        """deactivate_elements(missing, 'missing_data') as the first of the step's deactivations.  The reference's deactivate_outside
        that follows names its category as soon as ANY element lies beyond a drift:deactivate_*_of limit (:1774-1781), also when
        all of them have just been labelled 'missing_data' and keep that label; the housekeeping launch only looks at active
        elements, so that case is numbered here."""
        torch = self.engine.torch
        self.deactivate_elements(missing, reason='missing_data')
        if self.validity_domain is not None and 'outside' not in self.status_categories and bool(missing.any()):
            W, E, S, N = self.validity_domain
            lon, lat = self.elements.dev('lon', torch.float64), self.elements.dev('lat', torch.float64)
            if E is not None and E > 180 and bool((lon < 0).any()):
                lon = torch.where(lon < 0, lon + 360, lon)          # (:2359-2373)
            out = torch.zeros_like(missing)
            for lim, cmp_ in ((W, lambda a: lon < a), (E, lambda a: lon > a), (S, lambda a: lat < a), (N, lambda a: lat > a)):
                if lim is not None:
                    out |= cmp_(lim)
            if bool((out & missing).any()):
                self.status_categories.append('outside')

    def update_previous_state(self):
        """:642-669 for lon / lat (the element properties the reference stores when a coastline action may move elements back) and
        for sea_surface_height (the environment variable OceanDrift stores while vertical advection is on)."""
        if self.num_elements_active() == 0:
            return
        el, torch = self.elements, self.engine.torch
        if getattr(self, '_ssh_store', None) is not None:
            age = None
            if getattr(self, '_newly_seeded', False):              # newly_seeded_IDs is not None (:645-653)
                age = el.dev('age_seconds')
                if age.dtype not in (torch.float32, torch.float64):
                    age = age.to(torch.float64)
            self._ssh_prev = self.engine.store_previous_env(self._ssh_tensor(), el.dev('ID', torch.int32), age,
                                                            self.time_step.total_seconds(), self._id_base, self._ssh_store)
            self.environment_previous = EnvironmentView({'sea_surface_height': self._ssh_prev})
        if not getattr(self, '_store_previous', False):
            return
        self.engine.store_previous(el.dev('lon', torch.float64), el.dev('lat', torch.float64), el.dev('ID', torch.int32), self._id_base,
                                   self._prev_lon, self._prev_lat)

    # -- sea surface height (the water column is sea_floor_depth_below_sea_level + sea_surface_height) -----------------------
    def _vertical_advection_correction(self):
        return 'drift:vertical_advection_correction' in self._config and bool(self.get_config('drift:vertical_advection_correction'))

    def _ssh_reads(self):
        """Does anything in this run read the sea surface height per element?  (Overridden by OceanDrift.)"""
        return bool(self.env.priority_list.get('sea_floor_depth_below_sea_level'))

    def _setup_sea_level(self):
        """The previous-step store of sea_surface_height (required_variables store_previous_if, :1917-1924, :2162-2163: float32 per
        trajectory, NaN at the start) runs when its condition holds and the value can change -- a reader, a non-zero constant --
        or drift:vertical_advection_correction reads it.  A reader is sampled at the top of every step that something reads it in."""
        self._ssh_store = self._ssh_now = self._ssh_prev = None
        self.environment_previous = None
        self._ssh_sample_at_top = False
        spec = self.required_variables.get('sea_surface_height')
        if spec is None:
            return
        reader = bool(self.env.priority_list.get('sea_surface_height'))
        varies = reader or (self.env.constant('sea_surface_height') or 0) != 0
        cond = spec.get('store_previous_if')
        if cond is not None:
            key, op, val = cond
            cur = self.get_config(key)
            if ((op == 'is' and cur is val) or (op == 'in' and cur in val)) and (varies or self._vertical_advection_correction()):
                torch = self.engine.torch
                self._ssh_store = torch.full((len(self._release_rank),), float('nan'), dtype=torch.float32, device=self.engine.device)
        self._ssh_sample_at_top = reader and (self._ssh_store is not None or self._ssh_reads())

    def _sea_surface_height(self):
        """sea_surface_height at the elements at the start of the step: a float when no reader provides it (constant, else
        fallback), else the float32 device tensor."""
        if 'sea_surface_height' not in self.required_variables:
            return 0.0
        if not self.env.priority_list.get('sea_surface_height'):
            c = self.env.constant('sea_surface_height')
            if c is None:
                c = self.env.fallback('sea_surface_height')
            return float(c or 0.0)
        if getattr(self, '_ssh_now', None) is None:
            self._ssh_now = self._start_of_step_sample('sea_surface_height')
        return self._ssh_now

    def _ssh_tensor(self):
        s = self._sea_surface_height()
        if hasattr(s, 'data_ptr'):
            return s
        torch = self.engine.torch
        return torch.full((self.num_elements_active(),), float(np.float32(s)), dtype=torch.float32, device=self.engine.device)

    def _water_column(self, floor, tensor=False):
        """(sea floor, sea surface height) to hand to the kernels that compare depths with -(floor + ssh): with a per-element
        sea surface height, (floor + ssh as one float32 tensor -- NumPy's float32 sum --, 0.0); else (floor, the scalar ssh).
        tensor=True: a float32 tensor for the column whenever the sea surface height is not zero."""
        ssh = self._sea_surface_height()
        if not hasattr(ssh, 'data_ptr') and (ssh == 0 or not tensor):
            return floor, ssh
        torch = self.engine.torch
        if not hasattr(ssh, 'data_ptr'):
            ssh = self._ssh_tensor()
        if not hasattr(floor, 'data_ptr'):
            floor = torch.full_like(ssh, float(np.float32(floor)))
        return floor + ssh, 0.0

    def interact_with_seafloor(self):
        """:748-783 -- elements below the sea floor (sea_floor_depth_below_sea_level from a reader + sea_surface_height) are lifted
        to it, or lifted and deactivated ('seafloor'), as general:seafloor_action says; a no-op unless a reader provides the depth."""
        if self.num_elements_active() == 0 or not self.env.priority_list.get('sea_floor_depth_below_sea_level'):
            return
        action = self.get_config('general:seafloor_action')
        if action == 'none':
            return
        eng, el, torch = self.engine, self.elements, self.engine.torch
        floor, ssh = self._water_column(self._start_of_step_sample('sea_floor_depth_below_sea_level'))
        if action == 'previous':
            # elements below the floor go back to the horizontal position of the previous step, their depth stays (:775-783)
            lon, lat = el.dev('lon', torch.float64), el.dev('lat', torch.float64)
            eng.coastline(floor, lon, lat, self._z_for_sampling(), None, el.dev('status', torch.int32), el.dev('moving', torch.int32),
                          el.dev('ID', torch.int32), self._prev_lon, self._prev_lat, self._id_base, 'seafloor_previous', ssh=ssh)
            el.set_dev('lon', lon)
            el.set_dev('lat', lat)
            return
        z = self._z_for_sampling()
        code = 0
        if action == 'deactivate':
            # the category is numbered when the first element hits the floor; until then a provisional number is handed down
            code = self.status_categories.index('seafloor') if 'seafloor' in self.status_categories else len(self.status_categories)
        nd = eng.vertical_buoyancy(z, z, None, 0.0, sea_floor=floor, sea_surface_height=ssh, status=el.dev('status', torch.int32),
                                   moving=el.dev('moving', torch.int32), seafloor_code=code, count=code != 0)
        el.set_dev('z', z)
        if nd:
            if 'seafloor' not in self.status_categories:
                self.status_categories.append('seafloor')
            self._maybe_deactivated = True

    # -- environment ---------------------------------------------------------------------------------------
    def _active_variables(self):
        """Required variables after the skip_if conditionals (:1899-1924)."""
        out = []
        for v, spec in self.required_variables.items():
            cond = spec.get('skip_if')
            if cond is not None:
                key, op, val = cond
                cur = self.get_config(key)
                if (op == 'is' and cur is val) or (op == 'in' and cur in val):
                    continue
            out.append(v)
        return out

    @property
    def environment(self):
        """Start-of-step environment (float32 per variable), sampled lazily on the device."""
        if getattr(self, '_env_view', None) is None:
            el = self.elements
            d_env, missing = self.env.device_environment(self._env_variables, self.time, el.dev('lon', self.engine.torch.float64),
                                                         el.dev('lat', self.engine.torch.float64), self._z_truncated(),
                                                         pos_f32=el.positions_f32)
            self._add_uncertainty(d_env, stage0=True)
            self._env_view = EnvironmentView(d_env)
            self._env_missing = missing
        return self._env_view

    def _cover_elements_with_blocks(self):
        """Readers that hand out sub-blocks (reader_netCDF_CF_generic.py:404-626) are asked for the block around the elements, as
        StructuredReader does with the positions it is called with (structured.py:275-318): bounding box of the active elements
        (one reduction launch + a 32-byte read), grown by what an element can travel in one step at drift:max_speed.  The block is
        only replaced when the box has left the current one."""
        eng, el, torch = self.engine, self.elements, self.engine.torch
        bbox = eng.bbox(el.dev('lon', torch.float64), el.dev('lat', torch.float64))
        d = getattr(self, '_dist', None)
        if d is not None:                    # every rank must use the same window: the slabs are broadcast window-shaped
            bbox = d.allreduce_bbox(eng, bbox)
        lat_max = min(89.0, max(abs(bbox[2]), abs(bbox[3]))) if np.all(np.isfinite(bbox)) else 0.0
        margin = (self.get_config('drift:max_speed') * abs(self.time_step.total_seconds()) / (111000.0 * np.cos(np.radians(lat_max)))
                  + 1e-6)
        if any(self.env.ensure_windows(bbox, margin)):
            self._env_view = None

    def _start_of_step_sample(self, var):
        """float32 device tensor of ONE environment variable at the elements' current positions: from the step's environment when
        it has been materialised, else sampled on its own (the fused step never materialises the full environment)."""
        eng, el, torch = self.engine, self.elements, self.engine.torch
        if getattr(self, '_env_view', None) is not None and var in self._env_view:
            return self._env_view.dev(var, eng)
        d_env, _ = self.env.device_environment([var], self.time, el.dev('lon', torch.float64), el.dev('lat', torch.float64),
                                               self._z_truncated(), pos_f32=el.positions_f32)
        return d_env[var]

    def _uncertainty(self):
        return (self.get_config('drift:current_uncertainty', 0) or 0, self.get_config('drift:current_uncertainty_uniform', 0) or 0,
                self.get_config('drift:wind_uncertainty', 0) or 0)

    def _predraw_step_uncertainty(self):
        """The reference samples the step's environment -- and draws its uncertainty -- for every element that is active at the
        top of the loop, BEFORE deactivate_outside / retirement / removal (basemodel/__init__.py:2238-2262).  The draws of the
        legacy generator are therefore made here, for that element count, and follow the elements through the compaction."""
        self._noise0 = None
        cu, cuu, wu = self._uncertainty()
        n = self.num_elements_active()
        if n == 0 or not (cu > 0 or cuu > 0 or wu > 0):
            return
        d = {}
        if cu > 0:
            d['cur_n'] = [np.random.normal(0, cu, n), np.random.normal(0, cu, n)]
        if cuu > 0:
            d['cur_u'] = [np.random.uniform(-cuu, cuu, n), np.random.uniform(-cuu, cuu, n)]
        if wu > 0 and 'x_wind' in self._env_variables and 'y_wind' in self._env_variables:
            d['wind'] = [np.random.normal(0, wu, n), np.random.normal(0, wu, n)]
        self._noise0 = d

    def _add_uncertainty(self, d_env, stage0=False):
        """environment.py:869-891: env[var] += draw on float32 arrays.  stage0: the step's own environment, whose draws were
        made at the top of the loop (_predraw_step_uncertainty); otherwise (a Runge-Kutta stage) fresh draws."""
        cu, cuu, wu = self._uncertainty()
        eng, torch = self.engine, self.engine.torch
        n = self.num_elements_active()
        pre = getattr(self, '_noise0', None) if stage0 else None
        if pre is not None:
            def addp(var, draw):
                d_env[var] = (d_env[var].to(torch.float64) + eng.to_device(draw)).to(torch.float32)
            if 'x_sea_water_velocity' in d_env and 'y_sea_water_velocity' in d_env:
                for key in ('cur_n', 'cur_u'):
                    if key in pre:
                        addp('x_sea_water_velocity', pre[key][0])
                        addp('y_sea_water_velocity', pre[key][1])
            if 'x_wind' in d_env and 'y_wind' in d_env and 'wind' in pre:
                addp('x_wind', pre['wind'][0])
                addp('y_wind', pre['wind'][1])
            return

        def add(var, draw):
            d_env[var] = (d_env[var].to(torch.float64) + eng.to_device(draw)).to(torch.float32)
        if 'x_sea_water_velocity' in d_env and 'y_sea_water_velocity' in d_env:
            if cu > 0:
                add('x_sea_water_velocity', np.random.normal(0, cu, n))
                add('y_sea_water_velocity', np.random.normal(0, cu, n))
            if cuu > 0:
                add('x_sea_water_velocity', np.random.uniform(-cuu, cuu, n))
                add('y_sea_water_velocity', np.random.uniform(-cuu, cuu, n))
        if 'x_wind' in d_env and 'y_wind' in d_env and wu > 0:
            add('x_wind', np.random.normal(0, wu, n))
            add('y_wind', np.random.normal(0, wu, n))

    def _z_for_sampling(self):
        """Depth tensor in the dtype the reference's array has: float32, or float64 after vertical mixing."""
        z = self.elements.dev('z')
        if z.dtype not in (self.engine.torch.float32, self.engine.torch.float64):
            z = z.to(self.engine.torch.float64)
        return z

    def _z_truncated(self):
        """The depth the readers are asked at: drift:truncate_ocean_model_below_m (environment.py:554-562) clips a copy of z
        in its own dtype; the element depths themselves are untouched."""
        z = self._z_for_sampling()
        trunc = self.get_config('drift:truncate_ocean_model_below_m', None) \
            if 'drift:truncate_ocean_model_below_m' in self._config else None
        if trunc is None:
            return z
        torch = self.engine.torch
        return torch.where(z < -trunc, torch.full_like(z, -trunc), z)

    # -- positions (:4630-4669) ---------------------------------------------------------------------------------
    def update_positions(self, x_vel, y_vel):
        """Move particles with the given velocity components for one time step (WGS84 geodesic)."""
        eng, el = self.engine, self.elements
        torch = eng.torch
        xv = x_vel if isinstance(x_vel, torch.Tensor) else eng.to_device(np.ascontiguousarray(x_vel))
        yv = y_vel if isinstance(y_vel, torch.Tensor) else eng.to_device(np.ascontiguousarray(y_vel))
        if xv.dtype != yv.dtype or xv.dtype not in (torch.float32, torch.float64):
            xv, yv = xv.to(torch.float64), yv.to(torch.float64)
        moving = el.dev('moving')
        if moving.dtype != torch.int32:
            moving = moving.to(torch.int32)
        eng.update_positions(el.dev('lon', torch.float64), el.dev('lat', torch.float64), xv, yv, moving,
                             self.time_step.total_seconds())
        el.positions_f32 = False
        lon, lat = el.dev('lon'), el.dev('lat')
        # the reference aborts on invalid coordinates (:4661-4669); checked lazily at output steps here

    def _device_normals(self, n, k=2, salt=0):
        """k float64 device tensors of n standard-normal draws for the active elements.
        gpu:rng = numpy (default): np.random.normal of the legacy global generator, in the reference's order -- parity.
        gpu:rng = philox: drawn on the device from a generator keyed by (seed, step, salt) and indexed by element ID, so
        the draws do not depend on the order of the device arrays (which may then be re-sorted by cell) and nothing
        crosses the PCIe bus."""
        eng = self.engine
        torch = eng.torch
        if self.get_config('gpu:rng', 'numpy') != 'philox':
            return [eng.to_device(np.random.normal(scale=1, size=n)) for _ in range(k)]
        gen = torch.Generator(device=eng.device)
        gen.manual_seed((int(self._seed) * 1000003 + int(self.steps_calculation)) * 16 + int(salt))
        ids = self.elements.dev('ID').to(torch.int64)
        # (one value per element ID of the whole job, so that the draws do not depend on how the elements are sharded)
        n_ids = int(self.shard[2]) if getattr(self, 'shard', None) else int(self._id_base + self._n_total)
        base = torch.randn((k, n_ids), dtype=torch.float64, device=eng.device, generator=gen)
        return [base[j][ids] for j in range(k)]

    def horizontal_diffusion(self):
        """:1746-1772 -- two normal draws from the legacy global generator (x first), then update_positions."""
        if 'horizontal_diffusivity' not in self.required_variables or self.num_elements_active() == 0:
            return
        D = self._constant_or_none('horizontal_diffusivity')
        if D is None:
            D_dev = self.environment.dev('horizontal_diffusivity', self.engine)
            if float(D_dev.max()) == 0:
                return
        elif D == 0:
            return
        eng = self.engine
        n = self.num_elements_active()
        rx, ry = self._device_normals(n, 2, salt=1)
        dt = abs(self.time_step.total_seconds())
        torch = eng.torch
        if D is None:
            s = torch.sqrt(2 * D_dev / np.float32(dt))
        else:
            s = torch.full((n,), float(np.sqrt(np.float32(2) * np.float32(D) / np.float32(dt))), dtype=torch.float32,
                           device=eng.device)
        mv = self.elements.dev('moving').to(torch.float64)
        self.update_positions(mv * s.to(torch.float64) * rx, mv * s.to(torch.float64) * ry)

    def _constant_or_none(self, var):
        """Value of a variable that no reader provides (constant, else fallback), or None if a reader does."""
        c = self.env.constant(var)
        if c is not None:
            return c
        if not self.env.priority_list.get(var):
            return self.env.fallback(var)
        return None

    # -- the main loop (:1828-2340) -----------------------------------------------------------------------------
    def update(self):
        raise NotImplementedError('model subclasses implement update()')

    def update_and_diffuse(self):
        """One time step of the model physics (:2272-2280): update() then horizontal_diffusion()."""
        _ = self.environment          # sample the start-of-step environment before anything moves (:2238-2246)
        self.update()
        self.horizontal_diffusion()

    def prepare_run(self):
        pass

    def run(self, time_step=None, steps=None, time_step_output=None, duration=None, end_time=None,
            outfile=None, export_variables=None, export_buffer_length=100, stop_on_error=False):
        if outfile is not None:
            raise NotImplementedError('file export is outside the GPU hot path; read o.history / o.elements')
        if self.num_elements_scheduled() == 0:
            raise ValueError('Please seed elements before starting a run.')
        for key in ('drift:water_column_stretching', 'drift:use_tabularised_stokes_drift', 'vertical_mixing:TSprofiles'):
            if key in self._config and self.get_config(key):
                raise NotImplementedError('%s = True is not on the GPU path' % key)
        from .. import _lib
        self.engine.math_mode = {'series': _lib.OD_MATH_SERIES, 'exact': _lib.OD_MATH_EXACT,
                                 'fast': _lib.OD_MATH_FAST}[self.get_config('gpu:arithmetic')]
        if time_step is None:
            time_step = timedelta(minutes=self.get_config('general:time_step_minutes'))
        if not isinstance(time_step, timedelta):
            time_step = timedelta(seconds=time_step)
        self.time_step = time_step
        if time_step_output is None:
            tso = self.get_config('general:time_step_output_minutes')
            self.time_step_output = self.time_step if tso is None else timedelta(minutes=tso)
        else:
            self.time_step_output = time_step_output if isinstance(time_step_output, timedelta) \
                else timedelta(seconds=time_step_output)
            if self.time_step_output.days >= 0 and self.time_step.days < 0:
                self.time_step_output = -self.time_step_output
        ratio = self.time_step_output.total_seconds() / self.time_step.total_seconds()
        if ratio < 1:
            raise ValueError('Output time step must be equal or larger than calculation time step.')
        if not float(ratio).is_integer():
            raise ValueError('Ratio of calculation and output time steps must be an integer - given ratio is %s' % ratio)
        if time_step.days < 0:
            self.start_time = self.elements_scheduled_time.max()
        if sum(x is not None for x in (duration, end_time, steps)) > 1:
            raise ValueError('Only one of "steps", "duration" and "end_time" may be provided simultaneously')
        if duration is None and end_time is None:
            if steps is not None:
                duration = steps * self.time_step
            else:
                for r in self.env.readers.values():
                    if getattr(r, 'end_time', None) is not None:
                        end_time = r.end_time if end_time is None else min(end_time, r.end_time)
        if duration is None:
            duration = end_time - self.start_time
        if time_step.days < 0 and duration.days >= 0:
            duration = -duration
        if np.sign(duration.total_seconds()) * np.sign(time_step.total_seconds()) < 0:
            raise ValueError('Time step must be negative if duration is negative.')
        r = duration / self.time_step_output
        if not float(r).is_integer():
            duration = np.ceil(r) * self.time_step_output
        self.expected_steps_output = int(duration.total_seconds() / self.time_step_output.total_seconds() + 1)
        self.expected_steps_calculation = int(duration.total_seconds() / self.time_step.total_seconds())
        self.expected_end_time = self.start_time + self.expected_steps_calculation * self.time_step
        W, E = self.get_config('drift:deactivate_west_of'), self.get_config('drift:deactivate_east_of')
        S, N = self.get_config('drift:deactivate_south_of'), self.get_config('drift:deactivate_north_of')
        self.validity_domain = None if all(v is None for v in (W, E, S, N)) else [W, E, S, N]

        eng = self.engine
        self.env.finalize(eng)
        self._env_variables = [v for v in self._active_variables()
                               if self.env.priority_list.get(v) or self.env.constant(v) is not None
                               or self.env.fallback(v) is not None]
        self.elements = DeviceElements(self.ElementType, eng)
        self.time = self.start_time
        if self.time_step.days < 0:
            # 'Flipping ID array, so that lowest IDs are released first' (:2056-2062): in a backward run the element that
            # was scheduled last becomes ID 0 (IDs label the trajectories of the result)
            self.elements_scheduled.ID = np.flipud(np.asarray(self.elements_scheduled.ID))
        # A distributed run (torchrun, one process per GPU): every rank ran the same script and scheduled the same elements; each
        # keeps a contiguous index range of them (SURVEY 8(e): particle-index shards, replicated forcing).  Element IDs stay
        # global.  gpu:shard = none: the script seeded only this rank's elements itself.
        eng = self.engine
        eng.direction = -1 if self.time_step.days < 0 else 1
        if getattr(eng, 'dist', None) is None and self.get_config('gpu:distributed') and hasattr(eng, 'enable_distributed'):
            eng.enable_distributed()
        self._dist = getattr(eng, 'dist', None)
        if self._dist is not None and self._vertical_advection_correction():
            # the reference's previous-step store writes newly released elements at their positions in the whole element array
            # (update_previous_state :651-653); a shard sees only its own positions
            raise NotImplementedError('drift:vertical_advection_correction = True is not on the distributed GPU path')
        self.shard = None
        if self._dist is not None and self.get_config('gpu:shard') == 'index':
            n_all = int(self.num_elements_total())
            lo, hi = self._dist.shard(n_all)
            drop = np.ones(n_all, dtype=bool)
            drop[lo:hi] = False
            self.elements_scheduled.move_elements(self.ElementType(), drop)
            self.elements_scheduled_time = self.elements_scheduled_time[~drop]
            self.shard = (lo, hi, n_all)
        ids_all = np.atleast_1d(np.asarray(self.elements_scheduled.ID))
        self._id_base = int(ids_all.min()) if len(ids_all) else 0         # rows of the output block / rank table: ID - _id_base
        self._release_rank = np.full(int(ids_all.max()) - self._id_base + 1 if len(ids_all) else 0, -1, dtype=np.int64)
        self._released = 0
        self.steps_calculation = 0
        self._maybe_deactivated = False
        self._setup_coastline()
        self._setup_sea_level()
        if self.env.has_ensembles():
            ok = getattr(self, '_ensemble_variables', ())
            bad = [v for v in self.env.priority_list if self.env.has_ensembles([v]) and v not in ok]
            if bad:
                raise NotImplementedError('ensemble blocks for %s are not on the GPU path of %s' % (bad, type(self).__name__))
        out_every = int(round(ratio))
        n_total = len(self._release_rank)
        self._n_total = n_total
        self._out_every = out_every
        self._init_history(export_buffer_length)
        self.prepare_run()

        i = 0
        dist_run = self._dist is not None
        self._has_subblock_readers = bool(self.env.subblock_readers())
        # The step loop allocates small Python objects (argument structs, tensor handles) at a steady rate; a full collection of the
        # interpreter's cyclic garbage collector over everything the process has imported takes 50-150 ms -- the time of fifty
        # steps -- whenever it triggers.  The objects alive now are moved out of the collector's reach for the duration of the
        # loop (they stay reference-counted); what the loop allocates is still collected, in microseconds.
        import gc
        frozen = gc.isenabled()
        if frozen:
            gc.freeze()
        try:
            for i in range(self.expected_steps_calculation):
                self.release_elements()
                if dist_run:
                    # the slab collectives of this step, on every rank alike (also one that holds no elements right now)
                    self.env.touch_slabs(self._stage_times(self.time))
                if self.num_elements_active() == 0 and (self.num_elements_scheduled() > 0 or dist_run):
                    self.steps_calculation += 1                # (state_to_buffer with no elements: the column keeps its fill values)
                    self.time = self.time + self.time_step
                    continue
                self._env_view = None
                if self._has_subblock_readers:
                    self._cover_elements_with_blocks()
                self._ssh_now = None
                if self._ssh_sample_at_top:
                    # sampled with the step's environment, before anything moves the elements (:2238-2256)
                    self._ssh_now = self._start_of_step_sample('sea_surface_height')
                self._predraw_step_uncertainty()
                # deactivate_outside -> interact_with_seafloor -> state_to_buffer -> increase_age_and_retire (:2249-2260)
                col, only_deact = self._column_of_step(i)
                pm = getattr(self, '_pending_missing_code', None)
                if pm is not None:               # (Leeway with a coastline action: was the provisional 'missing_data' number used?)
                    self._pending_missing_code = None
                    if 'missing_data' not in self.status_categories and bool((self.elements.dev('status') == pm).any()):
                        self.status_categories.append('missing_data')
                self.report_missing_variables()                # (:2249, before deactivate_outside)
                if self._coast is not None:
                    # deactivate_outside -> interact_with_coastline -> interact_with_seafloor -> state_to_buffer -> ... (:2249-2260)
                    if self.env.priority_list.get('sea_floor_depth_below_sea_level'):
                        _ = self.environment                   # sampled before the lift, as the reference does (:2238-2256)
                    self._bookkeep(outside=True, age=False)
                    self.interact_with_coastline()
                    if self.env.priority_list.get('sea_floor_depth_below_sea_level'):
                        self.interact_with_seafloor()
                    self._bookkeep(outside=False, buffer_col=col, only_deactivated=only_deact, age=True)
                elif self.env.priority_list.get('sea_floor_depth_below_sea_level'):
                    _ = self.environment                       # sampled before the lift, as the reference does (:2238-2256)
                    self._bookkeep(outside=True, age=False)
                    self.interact_with_seafloor()
                    self._bookkeep(outside=False, buffer_col=col, only_deactivated=only_deact, age=True)
                else:
                    self._bookkeep(outside=True, buffer_col=col, only_deactivated=only_deact, age=True)
                self.remove_deactivated_elements()
                self.update_previous_state()                   # (:2262: positions elements may be moved back to)
                if self.num_elements_active() > 0:
                    self._maybe_sort()
                    self.update_and_diffuse()
                elif self.num_elements_scheduled() == 0 and not dist_run:
                    break                                      # 'No more active or scheduled elements' (:2276-2278): time is not advanced
                self.time = self.time + self.time_step
                self.steps_calculation += 1
        finally:
            if frozen:
                gc.unfreeze()
        self._env_view = None
        self.interact_with_coastline(final=True)           # (:2310)
        self._restore_id_order()
        self.state_to_buffer(final=True)
        self.remove_deactivated_elements()
        eng.sync()
        self._check_positions()
        self.result = self.history
        return self.history

    def _check_positions(self):
        """:4661-4669 -- the reference exits on invalid coordinates; raised here after the run."""
        if self.num_elements_active() == 0:
            return
        lon, lat = self.elements.dev('lon'), self.elements.dev('lat')
        lo, hi, ao, ai = float(lon.min()), float(lon.max()), float(lat.min()), float(lat.max())
        # (NaN compares False with everything: test for the valid range, not for the invalid one)
        if not (lo >= -180 and hi <= 360 and ao >= -90 and ai <= 90):
            if self._variables_that_may_miss() and not (lo < -180 or hi > 360 or ao < -90 or ai > 90):
                # Undefined positions are the reference's own outcome when a variable has no fallback value: a Runge-Kutta stage
                # outside the readers' coverage gives an undefined velocity, the element is taken out as 'missing_data' at the top of
                # the next step (the reference's check compares minima and maxima, which NaN passes, :4661-4669)
                return
            raise ValueError('Invalid new coordinates')

    def _restore_id_order(self):
        """Put the device arrays back in the reference's element order: the order of release (elements are appended as
        they are released and compaction is stable, elements.py:197-228), which is increasing ID only when the release
        times are monotonic in the seeding order of a forward run."""
        if not getattr(self, '_sorted', False) or self.num_elements_active() == 0:
            return
        torch = self.engine.torch
        ids = self.elements.dev('ID').to(torch.int64)
        key = self.engine.to_device(self._release_rank)[ids - self._id_base]
        perm = torch.argsort(key, stable=True).to(torch.int32)
        self.elements.permute(perm)
        self._sorted = False

    def _draws_follow_element_order(self):
        """True when this step consumes draws of NumPy's legacy generator element by element (parity mode): the device arrays
        must then stay in the reference's order.  Model classes add their own draws (vertical mixing, Leeway's jibing)."""
        if any(x > 0 for x in self._uncertainty()):
            return True   # the uncertainty draws are always the legacy generator's
        if self.get_config('gpu:rng', 'numpy') == 'philox':
            return False
        D = self._constant_or_none('horizontal_diffusivity') if 'horizontal_diffusivity' in self.required_variables else 0
        return D is None or D != 0

    def _maybe_sort(self):
        """Keep the device arrays ordered by grid cell (locality of the field gathers).  Element order is
        an implementation detail of the device arrays: outputs are keyed by ID."""
        k = self.get_config('gpu:sort_interval_steps')
        if not k or self.steps_calculation % k != 0 or self.num_elements_active() < 100000:
            return
        if self._draws_follow_element_order():
            return        # the legacy generator's draws are consumed in element order: keep the reference's order
        r = self.env.reader_for('x_sea_water_velocity', self.time)
        if r is None or not hasattr(r, 'group_of'):
            return
        g, _ = r.group_of('x_sea_water_velocity')
        el = self.elements
        t = self.engine.torch
        perm = self.engine.sort_by_cell(g, el.dev('lon', t.float64), el.dev('lat', t.float64), self._z_for_sampling())
        el.permute(perm)
        self._sorted = True
        if getattr(self, '_env_view', None) is not None:
            # the start-of-step environment follows the elements: sampling it again would see depths the sea-floor interaction
            # has already lifted (the reference samples once, before it, :2238-2256)
            self._env_view.permute(perm, self.engine)
        if getattr(self, '_ssh_now', None) is not None:
            self._ssh_now = self.engine.permute(perm, self._ssh_now)
        if getattr(self, '_ssh_prev', None) is not None:
            self._ssh_prev = self.engine.permute(perm, self._ssh_prev)
            self.environment_previous = EnvironmentView({'sea_surface_height': self._ssh_prev})

    # -- the output buffer (:2100-2135, 2384-2499) -----------------------------------------------------------------------
    # The reference pre-allocates result[var][trajectory, time] for the expected output times, NaN-filled; output steps write
    # every active element into the column of their time, sub-steps between output times write only the elements that were
    # deactivated, into the NEXT output column ('backfill'); the final state is written the same way and the time axis is cut at
    # the last time reached.  Here a block of columns [time][trajectory] lives in HBM (bounded: export_buffer_length columns and
    # gpu:history_block_bytes), filled by the bookkeeping launch and read back -- one contiguous copy per variable -- when the
    # next column falls outside the block.
    def _init_history(self, export_buffer_length):
        n_out = int(self.expected_steps_output)
        self._out_times = [self.start_time + k * self.time_step_output for k in range(n_out)]
        self.history = Result({'time': [], 'lon': [], 'lat': [], 'z': [], 'status': []})
        self.history.status_categories = self.status_categories
        per_col = 16 * max(1, int(self._n_total))
        cap = max(1, int(self.get_config('gpu:history_block_bytes')) // per_col)
        length = n_out if export_buffer_length is None else max(1, int(export_buffer_length))
        if self.get_config('gpu:history') == 'host':
            length = 1                                     # every output column goes to the host as soon as the next one starts
        self._hist_ncols = max(1, min(length, n_out, cap))
        self._hist_base = 0
        self._hist_dev = None
        self._hist_hi = -1                                 # highest column written so far
        # Long outputs (more columns than one device block): the host side of the buffer is page-locked memory for the whole
        # time axis, the device side two blocks used in turn, and a full block travels on the copy stream -- straight into its
        # final rows, no staging, no host copies -- while the steps go on writing the other block.
        eng = self.engine
        self._hist_pinned = None
        total = per_col * n_out
        if (n_out > self._hist_ncols and getattr(eng.device, 'type', 'cpu') == 'cuda' and total <= int(self.get_config('gpu:history_pinned_bytes'))
                and hasattr(eng, 'begin_copy_stream')):
            torch = eng.torch
            shape = (n_out, int(self._n_total))
            self._hist_pinned = tuple(torch.empty(shape, dtype=torch.float32, pin_memory=True) for _ in range(3)) + (
                torch.empty(shape, dtype=torch.int32, pin_memory=True),)
            self._hist_other, self._hist_other_ready = None, None

    def _column_of_step(self, i):
        """(output column, only_deactivated) of calculation step i: its own column on output steps, else the next one."""
        if i % self._out_every == 0:
            return i // self._out_every, False
        return i // self._out_every + 1, True

    def _new_hist_block(self):
        eng, torch = self.engine, self.engine.torch
        shape = (self._hist_ncols, int(self._n_total))
        return tuple(torch.full(shape, float('nan'), dtype=torch.float32, device=eng.device) for _ in range(3)) + (
            torch.full(shape, -1, dtype=torch.int32, device=eng.device),)

    def _hist_column(self, k):
        """The four device arrays [n_total] of output column k (flushing the block to the host when k lies beyond it)."""
        if self._hist_dev is None:
            self._hist_dev = self._new_hist_block()
        while k >= self._hist_base + self._hist_ncols:
            self._flush_history(self._hist_ncols)
        self._hist_hi = max(self._hist_hi, k)
        return tuple(b[k - self._hist_base] for b in self._hist_dev)

    def _flush_history(self, ncols):
        """Move the first ncols columns of the device block to the host side of the buffer."""
        if ncols <= 0:
            return
        h = self.history
        eng = self.engine
        if self._hist_pinned is not None and self._hist_dev is not None:
            # asynchronous: the block is copied into its rows of the page-locked buffer on the copy stream (which first waits for
            # the launches that filled it), reset there, and becomes the spare block; the steps continue on the other one
            base = self._hist_base
            if eng.begin_copy_stream():
                try:
                    for src, dst in zip(self._hist_dev, self._hist_pinned):
                        dst[base:base + ncols].copy_(src[:ncols], non_blocking=True)
                    for bq in self._hist_dev[:3]:
                        bq.fill_(float('nan'))
                    self._hist_dev[3].fill_(-1)
                finally:
                    ready = eng.end_copy_stream()
                spare, spare_ready = self._hist_other, self._hist_other_ready
                self._hist_other, self._hist_other_ready = self._hist_dev, ready
                if spare is None:
                    spare = self._new_hist_block()
                elif spare_ready is not None:
                    eng.wait_event(spare_ready)            # (a copy that finished long ago)
                self._hist_dev = spare
                for j in range(ncols):
                    h['time'].append(self._out_times[base + j])
                    for key, c in zip(('lon', 'lat', 'z', 'status'), self._hist_pinned):
                        h[key].append(c[base + j].numpy())     # (valid once the run has synchronised: run() does before it returns)
                self._hist_base += ncols
                return
        if self._hist_dev is None:
            cols = [np.full((ncols, int(self._n_total)), np.nan, dtype=np.float32) for _ in range(3)] + [
                np.full((ncols, int(self._n_total)), -1, dtype=np.int32)]
        elif self._hist_pinned is not None:
            base = self._hist_base
            for src, dst in zip(self._hist_dev, self._hist_pinned):
                dst[base:base + ncols].copy_(src[:ncols])
            cols = [c[base:base + ncols].numpy() for c in self._hist_pinned]
            for bq in self._hist_dev[:3]:
                bq.fill_(float('nan'))
            self._hist_dev[3].fill_(-1)
        else:
            # one device-to-host copy per variable (a host tensor -- the CPU tests -- shares its memory with the block: clone)
            cols = [(bq[:ncols].cpu() if bq.is_cuda else bq[:ncols].clone()).numpy() for bq in self._hist_dev]
            for bq in self._hist_dev[:3]:
                bq.fill_(float('nan'))
            self._hist_dev[3].fill_(-1)
        for j in range(ncols):
            h['time'].append(self._out_times[self._hist_base + j])
            for key, c in zip(('lon', 'lat', 'z', 'status'), cols):
                h[key].append(c[j])
        self._hist_base += ncols

    def state_to_buffer(self, final=False):
        """:2384-2403 for the current time; with final=True also the cut of the time axis at the time reached (:2425-2430)."""
        i = self.steps_calculation
        if self.num_elements_active() > 0:
            col, only_deact = self._column_of_step(i)
            if col < len(self._out_times):
                self._bookkeep(outside=False, buffer_col=col, only_deactivated=only_deact, age=False)
        if final:
            n_keep = i // self._out_every + 1              # output times <= the time reached
            while self._hist_base < n_keep:
                self._flush_history(min(self._hist_ncols, n_keep - self._hist_base))
            for key in self.history:
                del self.history[key][n_keep:]
            self._hist_dev = None
            if self._hist_pinned is not None:
                self.engine.order_after_copies()
                self._hist_other = None

    # -- small services model subclasses written for the reference call from update() -----------------------------------------
    def timer_start(self, category):
        """timer.py:26-34 (Timeable): wall-clock time per named category, e.g. 'main loop:updating elements:vertical mixing'.
        The launches are asynchronous: a category holds the time its host code took, not the time of the kernels it started."""
        from datetime import datetime as _dt
        self.__dict__.setdefault('timing', {}).setdefault(category, timedelta(0))
        self.__dict__.setdefault('timers', {})[category] = _dt.now()

    def timer_end(self, category):
        from datetime import datetime as _dt
        t0 = self.__dict__.setdefault('timers', {}).get(category)
        if t0 is not None:
            self.__dict__.setdefault('timing', {})[category] = self.__dict__['timing'].get(category, timedelta(0)) + (_dt.now() - t0)
        self.timers[category] = None

    def performance(self):
        """basemodel/__init__.py:809-836: the categories of timer_start / timer_end, indented by their ':' levels."""
        out = '--------------------\nPerformance:\n'
        for category, t in self.__dict__.get('timing', {}).items():
            parts = category.split(':')
            out += '%s%7.1f %s\n' % ('  ' * (len(parts) - 1), t.total_seconds(), parts[-1].replace('<colon>', ':'))
        return out + '--------------------\n'

    def store_message(self, message):
        """:4736-4740"""
        self.__dict__.setdefault('messages', []).append(message)

    def get_messages(self):
        return ''.join('%s\n' % m for m in self.__dict__.get('messages', []))

    def water_column_stretching(self):
        """oceandrift.py:299-313: a no-op unless drift:water_column_stretching is on -- which needs the previous sea surface height and
        is refused when the run starts (DESIGN.md row a14); here so that an update() written for the reference can call it."""
        if 'drift:water_column_stretching' in self._config and self.get_config('drift:water_column_stretching'):
            raise NotImplementedError('drift:water_column_stretching = True is not on the GPU path')

    def get_lonlats(self):
        return np.array(self.history['lon']).T, np.array(self.history['lat']).T

    def elements_by_id(self):
        """Active elements' lon/lat/z ordered by ID (the device arrays may be cell-sorted)."""
        el = self.elements
        ids = el.to_host_array('ID').astype(np.int64)
        order = np.argsort(ids, kind='stable')
        return (ids[order], el.to_host_array('lon')[order], el.to_host_array('lat')[order],
                el.to_host_array('z')[order])
