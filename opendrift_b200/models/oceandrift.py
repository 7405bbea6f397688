"""OceanDrift on the GPU hot path: the reference's model class (opendrift/models/oceandrift.py) with the same
element type, required variables, configuration keys and update() recipe for the advection path:

    update():  advect_ocean_current -> advect_wind -> stokes_drift -> vertical_advection      (:185-211)
    then the run loop's horizontal_diffusion                                                   (basemodel :2280)

When update() is not overridden by a subclass the whole recipe runs as ONE kernel launch per time step
(od_step_oceandrift); a subclass that overrides update() gets the same helpers as separate launches.
Vertical turbulent mixing (:397-571) runs as one extra launch per step (od_vertical_mixing, all inner iterations fused).
"""
import numpy as np

from ..config import CONFIG_LEVEL_ESSENTIAL, CONFIG_LEVEL_BASIC, CONFIG_LEVEL_ADVANCED
from ..elements import LagrangianArray
from .basemodel import OpenDriftSimulation


class Lagrangian3DArray(LagrangianArray):
    """oceandrift.py:28-51"""
    variables = LagrangianArray.add_variables([
        ('wind_drift_factor', {'dtype': np.float32, 'units': '1', 'default': 0.02,
                               'description': 'Elements at surface are moved with this fraction of the wind vector'}),
        ('current_drift_factor', {'dtype': np.float32, 'units': '1', 'default': 1,
                                  'description': 'Elements are moved with this fraction of the current vector'}),
        ('terminal_velocity', {'dtype': np.float32, 'units': 'm/s', 'default': 0.,
                               'description': 'Terminal rise/sinking velocity (buoyancy)'})])


class OceanDrift(OpenDriftSimulation):
    ElementType = Lagrangian3DArray
    _coast_previous_supported = True      # update() can run from the materialised start-of-step environment (helper recipe)
    # variables whose reader may serve ensemble blocks (member = i % n_members): sampled through Reader.sample_groups by the helper recipes
    _ensemble_variables = ('x_sea_water_velocity', 'y_sea_water_velocity', 'x_wind', 'y_wind', 'upward_sea_water_velocity',
                           'sea_surface_wave_stokes_drift_x_velocity', 'sea_surface_wave_stokes_drift_y_velocity',
                           'sea_surface_wave_significant_height', 'horizontal_diffusivity')

    # oceandrift.py:70-92
    required_variables = {
        'x_sea_water_velocity': {'fallback': 0},
        'y_sea_water_velocity': {'fallback': 0},
        'x_wind': {'fallback': 0},
        'y_wind': {'fallback': 0},
        'upward_sea_water_velocity': {'fallback': 0, 'skip_if': ['drift:vertical_advection', 'is', False]},
        'ocean_vertical_diffusivity': {'fallback': 0, 'skip_if': ['drift:vertical_mixing', 'is', False], 'profiles': True},
        'horizontal_diffusivity': {'fallback': 0},
        'sea_surface_wave_significant_height': {'fallback': 0},
        'sea_surface_wave_stokes_drift_x_velocity': {'fallback': 0, 'skip_if': ['drift:stokes_drift', 'is', False]},
        'sea_surface_wave_stokes_drift_y_velocity': {'fallback': 0, 'skip_if': ['drift:stokes_drift', 'is', False]},
        'ocean_mixed_layer_thickness': {'fallback': 50, 'skip_if': ['drift:vertical_mixing', 'is', False]},
        'sea_floor_depth_below_sea_level': {'fallback': 10000},
        'sea_surface_height': {'fallback': 0, 'store_previous_if': ['drift:vertical_advection', 'is', True]},
        'land_binary_mask': {'fallback': None},
    }

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._add_config({
            'drift:vertical_advection': {'type': 'bool', 'default': True, 'level': CONFIG_LEVEL_ESSENTIAL,
                                         'description': 'Advect elements with vertical component of ocean current.'},
            'drift:vertical_advection_at_surface': {'type': 'bool', 'default': False, 'level': CONFIG_LEVEL_ADVANCED,
                                                    'description': 'Also advect elements at the surface vertically.'},
            'drift:vertical_mixing': {'type': 'bool', 'default': False, 'level': CONFIG_LEVEL_BASIC,
                                      'description': 'Activate vertical mixing scheme with inner loop'},
            'drift:vertical_mixing_at_surface': {'type': 'bool', 'default': False, 'level': CONFIG_LEVEL_ADVANCED,
                                                 'description': 'Surface elements (z=0) are only mixed if True.'},
            'vertical_mixing:timestep': {'type': 'float', 'min': 0.1, 'max': 3600, 'default': 60, 'units': 'seconds',
                                         'level': CONFIG_LEVEL_ADVANCED,
                                         'description': 'Time step used for inner loop of vertical mixing.'},
            'vertical_mixing:diffusivitymodel': {'type': 'enum', 'default': 'environment',
                                                 'enum': ['environment', 'stepfunction', 'windspeed_Sundby1983',
                                                          'windspeed_Large1994', 'constant'],
                                                 'level': CONFIG_LEVEL_ADVANCED,
                                                 'description': 'Algorithm/source used for profile of vertical diffusivity. '
                                                                'Environment means that diffusivity is aquired from '
                                                                'readers or environment constants/fallback.'},
            'vertical_mixing:background_diffusivity': {'type': 'float', 'min': 0, 'max': 1, 'default': 1.2e-5,
                                                       'level': CONFIG_LEVEL_ADVANCED, 'units': 'm2s-1', 'description':
                                                       'Background diffusivity used below mixed layer for wind parameterisations.'},
            'drift:water_column_stretching': {'type': 'bool', 'default': False, 'level': CONFIG_LEVEL_ADVANCED,
                                              'description': 'Accepted with the reference\'s default; True is refused at run().'},
            'drift:vertical_advection_correction': {'type': 'bool', 'default': False, 'level': CONFIG_LEVEL_ADVANCED,
                                                    'description': 'Subtract the vertical motion of the water due to the change in '
                                                                   'sea surface height from the vertical water velocity '
                                                                   '(refused in distributed runs).'},
            'drift:use_tabularised_stokes_drift': {'type': 'bool', 'default': False, 'level': CONFIG_LEVEL_BASIC,
                                                   'description': 'Accepted with the reference\'s default; True is refused at run().'},
            'drift:tabularised_stokes_drift_fetch': {'type': 'enum', 'enum': ['5000', '25000', '50000'], 'default': '25000',
                                                     'level': CONFIG_LEVEL_ADVANCED, 'description': 'Only used with tabularised Stokes drift.'},
            'vertical_mixing:TSprofiles': {'type': 'bool', 'default': False, 'level': CONFIG_LEVEL_ADVANCED,
                                           'description': 'Accepted with the reference\'s default; True is refused at run().'},
            'gpu:rng': {'type': 'enum', 'enum': ['numpy', 'philox'], 'default': 'numpy', 'level': CONFIG_LEVEL_ADVANCED,
                        'description': 'numpy: draws of the legacy global generator made on the host in the reference\'s '
                                       'order (bit parity); philox: counter-based generator on the device keyed by element ID.'},
            'drift:stokes_drift': {'type': 'bool', 'default': True, 'level': CONFIG_LEVEL_ADVANCED,
                                   'description': 'Advection elements with Stokes drift (wave orbital motion).'},
            'drift:stokes_drift_profile': {'type': 'enum', 'default': 'Phillips',
                                           'enum': ['monochromatic', 'exponential', 'Phillips', 'windsea_swell'],
                                           'level': CONFIG_LEVEL_ADVANCED,
                                           'description': 'Algorithm to calculate Stokes drift at depth from surface value'},
            'drift:wind_drift_depth': {'type': 'float', 'default': 0.1, 'min': 0, 'max': 10, 'units': 'meters',
                                       'level': CONFIG_LEVEL_ADVANCED,
                                       'description': 'Wind drift decreases linearly to zero at this depth.'},
            'drift:truncate_ocean_model_below_m': {'type': 'float', 'default': None, 'min': 0, 'max': 10000,
                                                   'units': 'm', 'level': CONFIG_LEVEL_ADVANCED,
                                                   'description': 'Ocean model data are only read down to this depth.'},
        })
        self._set_config_default('drift:max_speed', 2)

    # -- the reference recipe, helper by helper (used when a subclass overrides update()) -------------------
    def update(self):
        self.advect_ocean_current()
        self.advect_wind()
        self.stokes_drift()
        self.update_terminal_velocity()
        if self.get_config('drift:vertical_mixing'):
            self.vertical_mixing()
        else:
            self.vertical_buoyancy()
        self.vertical_advection()

    def update_terminal_velocity(self, *args, **kwargs):
        """oceandrift.py:213-222: a hook for subclasses (plankton, oil droplets ...); the stock model keeps the seeded values."""
        pass

    # -- per-iteration hooks of the mixing loop (oceandrift.py:369-379): no-ops here, overridden by e.g. oil and plankton models --
    def prepare_vertical_mixing(self):
        pass

    def surface_stick(self):
        """Elements above the surface are put back onto it (the mixing launch does this itself unless a subclass overrides it)."""
        el, torch = self.elements, self.engine.torch
        z = self._z_for_sampling()
        el.set_dev('z', torch.clamp(z, max=0.0))

    def bottom_interaction(self, Zmin=None):
        pass

    def surface_wave_mixing(self, time_step_seconds):
        pass

    MIXING_HOOKS = ('prepare_vertical_mixing', 'update_terminal_velocity', 'surface_stick', 'surface_wave_mixing', 'bottom_interaction')

    def _overridden_mixing_hooks(self):
        return [h for h in self.MIXING_HOOKS if getattr(type(self), h) is not getattr(OceanDrift, h)]

    def _ssh_reads(self):
        """Readers of the per-element sea surface height besides the previous-step store: the sea floor (a reader for its depth),
        vertical mixing, drift:vertical_advection_correction, a bottom_interaction of a subclass (handed -(floor + ssh))."""
        return (super()._ssh_reads() or bool(self.get_config('drift:vertical_mixing')) or self._vertical_advection_correction()
                or type(self).bottom_interaction is not OceanDrift.bottom_interaction)

    def _buoyancy_inputs(self):
        """(sea floor tensor or None, sea_surface_height, status code for 'deactivate' or 0): the sea-floor part of
        vertical_buoyancy only acts when a reader provides the depth (interact_with_seafloor, basemodel/__init__.py:752-753).
        A per-element sea surface height comes added to the floor (the water column, float32)."""
        if not self.env.priority_list.get('sea_floor_depth_below_sea_level'):
            return None, 0.0, 0
        action = self.get_config('general:seafloor_action')
        if action == 'none':
            return None, 0.0, 0
        if action == 'previous':
            return None, 0.0, 0        # no lift: vertical_buoyancy() moves the elements below the floor back afterwards
        floor, ssh = self._water_column(self._start_of_step_sample('sea_floor_depth_below_sea_level'))
        code = 0
        if action == 'deactivate':
            code = self.status_categories.index('seafloor') if 'seafloor' in self.status_categories else len(self.status_categories)
        return floor, ssh, code

    def _buoyancy(self, z_in):
        """oceandrift.py:352-367 on the device (od_vertical_buoyancy): returns the new depth tensor (dtype of z_in)."""
        eng, el, torch = self.engine, self.elements, self.engine.torch
        tv = el.dev('terminal_velocity')
        if tv.dtype not in (torch.float32, torch.float64):
            tv = el.dev('terminal_velocity', torch.float64)
        floor, ssh, code = self._buoyancy_inputs()
        z_out = torch.empty_like(z_in)
        nd = eng.vertical_buoyancy(z_in, z_out, tv, self.time_step.total_seconds(), sea_floor=floor, sea_surface_height=ssh,
                                   status=el.dev('status', torch.int32), moving=el.dev('moving', torch.int32),
                                   seafloor_code=code, count=code != 0)
        if nd:
            if 'seafloor' not in self.status_categories:
                self.status_categories.append('seafloor')
            self._maybe_deactivated = True
        return z_out

    def vertical_buoyancy(self):
        """oceandrift.py:352-367: z[z < 0] = min(0, z + terminal_velocity * dt), then the sea floor."""
        self.elements.set_dev('z', self._buoyancy(self._z_for_sampling()))
        if self.get_config('general:seafloor_action') == 'previous' and self.env.priority_list.get('sea_floor_depth_below_sea_level'):
            self.interact_with_seafloor()          # (:363-366: elements that sank below the floor go back to their previous position)

    def vertical_advection(self):
        """oceandrift.py:315-350: z = min(0, z + moving*w*dt) below (or at) the surface; with drift:vertical_advection_correction
        w less the vertical motion of the water column due to the change of the sea surface height since the previous step."""
        if self.get_config('drift:vertical_advection') is False:
            return
        env = self.environment
        if 'upward_sea_water_velocity' not in env:
            return
        eng, el, torch = self.engine, self.elements, self.engine.torch
        w = env.dev('upward_sea_water_velocity', eng)
        if self._vertical_advection_correction() and getattr(self, '_ssh_prev', None) is not None:
            floor = self._constant_or_none('sea_floor_depth_below_sea_level')
            if floor is None:
                floor = env.dev('sea_floor_depth_below_sea_level', eng)
            z = self._z_for_sampling().clone()
            eng.vertical_advection_corrected(z, w, self._ssh_tensor(), self._ssh_prev, floor, el.dev('moving', torch.int32),
                                             self.get_config('drift:vertical_advection_at_surface'), self.time_step.total_seconds())
            el.set_dev('z', z)
            return
        z = el.dev('z')
        mv = el.dev('moving').to(torch.float64)
        ok = (z <= 0) if self.get_config('drift:vertical_advection_at_surface') else (z < 0)
        zn = torch.clamp(z.to(torch.float64) + mv * w.to(torch.float64) * self.time_step.total_seconds(), max=0.0)
        el.set_dev('z', torch.where(ok, zn.to(z.dtype), z))

    # -- vertical mixing (oceandrift.py:397-571) --------------------------------------------------------------------
    def _mixing_inputs(self):
        """Which diffusivity column the reference would use (oceandrift.py:425-453): the ocean-model profile when a
        gridded ocean_vertical_diffusivity reader serves this time, else Large et al. (1994) from the wind; or the
        analytical / constant model the configuration names."""
        model = self.get_config('vertical_mixing:diffusivitymodel')
        g = None
        if model == 'environment':
            r = self.env.reader_for('ocean_vertical_diffusivity', self.time)
            if len(self.env.readers_for('ocean_vertical_diffusivity', self.time)) > 1:
                raise NotImplementedError('vertical mixing on the GPU path takes its diffusivity profile from one reader; '
                                          'several readers provide ocean_vertical_diffusivity at %s' % self.time)
            if r is not None and hasattr(r, 'group_of'):
                g, _ = r.group_of('ocean_vertical_diffusivity')
            else:
                model = 'windspeed_Large1994'
        elif model not in ('windspeed_Large1994', 'windspeed_Sundby1983', 'constant'):
            raise NotImplementedError('vertical_mixing:diffusivitymodel = %r is not on the GPU path' % model)
        dt_mix = self.get_config('vertical_mixing:timestep') * np.sign(self.time_step.total_seconds())
        ntimes = int(np.abs(int(self.time_step.total_seconds() / dt_mix)))
        floor = self._constant_or_none('sea_floor_depth_below_sea_level')
        if floor is None:
            floor = self.environment.dev('sea_floor_depth_below_sea_level', self.engine)
        return g, model, dt_mix, ntimes, floor

    def _mixing_reads_environment(self):
        """True when the mixing launch needs start-of-step environment samples (wind for the analytical diffusivity models, a
        mixed-layer or sea-floor depth that comes from a reader) in addition to the diffusivity profile itself."""
        model = self.get_config('vertical_mixing:diffusivitymodel')
        if model == 'environment':
            r = self.env.reader_for('ocean_vertical_diffusivity', self.time)
            if r is None or not hasattr(r, 'group_of'):
                return True                           # falls back to Large et al. (1994): wind speed
        else:
            return True
        return self._constant_or_none('sea_floor_depth_below_sea_level') is None

    def _env_scalar_or_tensor(self, var, default):
        """A float (constant / fallback with no reader) or the start-of-step float32 device tensor of an environment variable."""
        c = self._constant_or_none(var)
        if c is not None:
            return float(c)
        if self.env.reader_for(var, self.time) is None:
            fb = self.env.fallback(var)
            return float(default if fb is None else fb)
        return self.environment.dev(var, self.engine)

    def _mix(self, lon0, lat0, z_in, pos_f32):
        """Run the mixing kernel from start-of-step positions; returns the new float64 depth tensor."""
        eng, el, torch = self.engine, self.elements, self.engine.torch
        g, model, dt_mix, ntimes, floor = self._mixing_inputs()
        # Zmin = -1.*(sea_floor_depth + sea_surface_height) (:420): the kernel negates the float32 column it is handed
        floor, _ = self._water_column(floor, tensor=True)
        n = len(el)
        moving = el.dev('moving')
        if moving.dtype != torch.int32:
            moving = moving.to(torch.int32)
        tv = el.dev('terminal_velocity') if 'terminal_velocity' in el.variables else None
        ids = el.dev('ID')
        if ids.dtype != torch.int32:
            ids = ids.to(torch.int32)
        kw = {}
        if model != 'environment':
            env = self.environment
            if 'x_wind' in env and 'y_wind' in env:
                xw, yw = env.dev('x_wind', eng), env.dev('y_wind', eng)
                ws = torch.sqrt(xw * xw + yw * yw)                                       # PhysicsMethods.wind_speed (:885-887)
            else:
                ws = torch.zeros(n, dtype=torch.float32, device=eng.device)
            kw = dict(model=model, wind_speed=ws,
                      mld=self._env_scalar_or_tensor('ocean_mixed_layer_thickness', 50.0),
                      background=self.get_config('vertical_mixing:background_diffusivity'),
                      k_const=float(self.env.fallback('ocean_vertical_diffusivity') or 0.0))
        # 'Let particles stick to bottom' (oceandrift.py:559-564) only acts when a reader provides the sea floor
        action, code, status = 0, 0, None
        if self.env.priority_list.get('sea_floor_depth_below_sea_level'):
            cfg = self.get_config('general:seafloor_action')
            if cfg == 'previous':
                raise NotImplementedError("general:seafloor_action = 'previous' is not on the GPU path")
            action = {'none': 0, 'lift_to_seafloor': 1, 'deactivate': 2}[cfg]
            if action == 2:
                cats = self.status_categories
                code = cats.index('seafloor') if 'seafloor' in cats else len(cats)
                status = el.dev('status', torch.int32)
                moving = el.dev('moving', torch.int32)
        common = dict(moving=moving, ids=ids, seed=getattr(self, '_seed', 0), step_index=self.steps_calculation, sea_floor=floor,
                      mix_at_surface=self.get_config('drift:vertical_mixing_at_surface'), pos_f32=pos_f32, **kw)
        hooks = self._overridden_mixing_hooks()
        if not hooks:
            # the whole inner loop in one launch
            rand = None
            if self.get_config('gpu:rng') == 'numpy':          # the reference's draws, in its order (:524)
                rand = eng.to_device(np.ascontiguousarray(np.stack([np.random.random(n) for _ in range(ntimes)])))
            z_out = eng.vertical_mixing(g, self.time, lon0, lat0, z_in, dt_mix, ntimes, terminal_velocity=tv, rand=rand,
                                        seafloor_action=action, status=status, seafloor_code=code, **common)
            if action == 2 and getattr(eng, 'last_mix_deactivated', 0):
                if 'seafloor' not in self.status_categories:
                    self.status_categories.append('seafloor')
                self._maybe_deactivated = True
            return z_out
        # A subclass overrides a per-iteration hook: one launch per inner iteration, the hooks in between, in the reference's
        # order (:515-564): [update_terminal_velocity] random walk + reflections + buoyancy [surface_stick] [surface_wave_mixing]
        # sea floor [bottom_interaction].  The draws of the legacy generator are made iteration by iteration, as the reference does
        # (a hook may draw too); the device generator continues its per-step stream (iter0).
        self.prepare_vertical_mixing()
        z = z_in
        numpy_rng = self.get_config('gpu:rng') == 'numpy'
        for it in range(ntimes):
            if 'update_terminal_velocity' in hooks:
                el.set_dev('z', z)
                self.update_terminal_velocity(Tprofiles=None, Sprofiles=None, z_index=None)
                tv = el.dev('terminal_velocity')
            r = eng.to_device(np.ascontiguousarray(np.random.random(n)[None])) if numpy_rng else None
            z = eng.vertical_mixing(g, self.time, lon0, lat0, z, dt_mix, 1, terminal_velocity=tv, rand=r, iter0=it,
                                    skip_surface_stick='surface_stick' in hooks, **common)
            el.set_dev('z', z)
            if 'surface_stick' in hooks:
                self.surface_stick()
            if 'surface_wave_mixing' in hooks:
                self.surface_wave_mixing(abs(dt_mix))
            # 'Let particles stick to bottom' (:557-561): which elements are below -(floor + ssh) is decided before
            # interact_with_seafloor lifts them; bottom_interaction then gets that Zmin
            below = False
            if 'bottom_interaction' in hooks:
                zmin = -(self.environment.sea_floor_depth_below_sea_level + self.environment.sea_surface_height) \
                    if 'sea_surface_height' in self.environment else -self.environment.sea_floor_depth_below_sea_level
                below = bool((np.asarray(el.z) < zmin).any())
            if action:
                self._stick_to_bottom(floor, action, code)
            if below:
                self.bottom_interaction(zmin)
            z = self._z_for_sampling()
        return z

    def _stick_to_bottom(self, floor, action, code):
        """interact_with_seafloor at the end of a mixing iteration (:559-563)."""
        eng, el, torch = self.engine, self.elements, self.engine.torch
        z = self._z_for_sampling()
        if not hasattr(floor, 'data_ptr'):
            return
        nd = eng.vertical_buoyancy(z, z, None, 0.0, sea_floor=floor, status=el.dev('status', torch.int32),
                                   moving=el.dev('moving', torch.int32), seafloor_code=code if action == 2 else 0, count=action == 2)
        el.set_dev('z', z)
        if nd:
            if 'seafloor' not in self.status_categories:
                self.status_categories.append('seafloor')
            self._maybe_deactivated = True

    def vertical_mixing(self, store_depths=False):
        """Helper for subclasses that override update(): uses the start-of-step positions saved by the run loop."""
        if self.get_config('drift:vertical_mixing') is False:
            return
        lon0, lat0, f32 = self._start_positions
        self.elements.set_dev('z', self._mix(lon0, lat0, self._z_for_sampling(), f32))

    def _draws_follow_element_order(self):
        if super()._draws_follow_element_order():
            return True
        # the mixing loop draws np.random.random(n) per inner iteration (oceandrift.py:524)
        return bool(self.get_config('drift:vertical_mixing')) and self.get_config('gpu:rng') == 'numpy'

    # -- fused path -----------------------------------------------------------------------------------------------
    def _fused_ok(self):
        t = type(self)
        return (t.update is OceanDrift.update and t.advect_ocean_current is OceanDrift.advect_ocean_current
                and t.vertical_mixing is OceanDrift.vertical_mixing and t.vertical_buoyancy is OceanDrift.vertical_buoyancy
                and t.update_terminal_velocity is OceanDrift.update_terminal_velocity
                and not self.get_config('drift:relative_wind'))
        # (overridden mixing hooks are served inside _mix: one launch per inner iteration)

    def run(self, *args, **kwargs):
        self._use_fused = None
        # does any element that this run will release have a buoyancy?  (decides whether the fused step needs the extra launch)
        self._tv_nonzero = False
        if hasattr(self, 'elements_scheduled') and 'terminal_velocity' in self.ElementType.variables:
            self._tv_nonzero = bool(np.any(np.atleast_1d(self.elements_scheduled.terminal_velocity) != 0))
        return super().run(*args, **kwargs)

    def _step_fused(self):
        eng, el, torch = self.engine, self.elements, self.engine.torch
        g = self._current_group(self.time)
        if g is None:
            return False
        if getattr(self, '_coast_moved', False):
            return False        # elements were moved back from land: they keep the environment sampled where they were (helper recipe)
        if self.env.has_ensembles():
            return False        # ensemble blocks: every sample goes through Reader.sample_groups (helper / staged recipes)
        if self.env.has_host_readers():
            return False        # a reader that computes its values on the host (readers/continuous.py): helper / staged recipes
        if self._vertical_advection_correction():
            return False        # the corrected vertical advection is a launch of its own after the moves (helper recipe)
        if self.env.priority_list.get('sea_floor_depth_below_sea_level'):
            # A reader for the sea floor: elements below it are lifted at the top of the loop, AFTER the step's environment was
            # sampled (basemodel/__init__.py:2238-2256) -- the first Runge-Kutta stage and w see the depth before the lift, the
            # later stages the depth after it.  The helper recipe does exactly that with the materialised environment.
            return False
        t = self.time
        chain = ()
        if self._current_needs_reader_loop(t):
            groups = self._current_chain(t)               # reader priority list inside the kernel, when it can be
            if groups is None:
                return False
            g, chain = groups[0], tuple(groups[1:])
        if any(len(self.env.readers_for(v, t)) > 1 for v in ('x_wind', 'y_wind', 'upward_sea_water_velocity')):
            return False                                  # several readers for one variable: the helpers loop over them
        wind_r = self.env.reader_for('x_wind', t)
        wind = wind_r.group_of('x_wind')[0] if wind_r is not None and hasattr(wind_r, 'group_of') else None
        if wind is not None and (wind.ncomp != 2 or self.env.reader_for('y_wind', t) is not wind_r):
            return False                                  # wind components from different sources: helper path
        if wind is None and (self._constant_or_none('x_wind') or 0) != 0:
            return False                                  # constant non-zero wind: helper path
        wgrp = None
        if self.get_config('drift:vertical_advection'):
            wr = self.env.reader_for('upward_sea_water_velocity', t)
            wgrp = wr.group_of('upward_sea_water_velocity')[0] if wr is not None and hasattr(wr, 'group_of') else None
            if wgrp is None and (self._constant_or_none('upward_sea_water_velocity') or 0) != 0:
                return False
        D = self._constant_or_none('horizontal_diffusivity')
        if D is None:
            return False                                  # gridded diffusivity: helper path
        # Stokes drift moves between wind drift and the random walk: when it is active its start-of-step samples
        # are taken first, the fused kernel does current + wind (+ w), then the Stokes and diffusion launches follow
        stokes_inp = None
        if self.get_config('drift:stokes_drift') and any(
                self.env.priority_list.get(v) or (self.env.constant(v) or 0) != 0
                for v in ('sea_surface_wave_stokes_drift_x_velocity', 'sea_surface_wave_stokes_drift_y_velocity')):
            stokes_inp = self._stokes_inputs()
        split_diffusion = stokes_inp is not None and D != 0
        n = len(el)
        from ..engine import draw_uncertainty
        cu, cuu, wu = self._uncertainty()
        if stokes_inp is not None and (cu > 0 or cuu > 0 or wu > 0):
            return False        # the step's environment (with its draws) is already materialised: helper path
        if wu > 0 and wind is None:
            return False        # the reference adds the wind uncertainty to the fallback wind too: helper path
        if (cu > 0 or cuu > 0 or wu > 0) and self.get_config('drift:vertical_mixing') and self._mixing_reads_environment():
            return False        # the mixing launch would materialise the environment and draw its uncertainty a second time
        ncur, nkinds, nwind = draw_uncertainty(n, self.get_config('drift:advection_scheme'), cu, cuu, wu,
                                               with_wind=wind is not None, stage0=getattr(self, '_noise0', None))
        d_ncur = eng.to_device(ncur) if ncur is not None else None
        d_nwind = eng.to_device(nwind) if nwind is not None else None
        moving = el.dev('moving')
        if moving.dtype != torch.int32:
            moving = moving.to(torch.int32)
        fac = el.dev('current_drift_factor')
        z = self._z_for_sampling()
        el.set_dev('z', z)
        z_new = None
        if self.get_config('drift:vertical_mixing'):
            # mixing first: it reads the start-of-step positions and depth and writes a new depth buffer; the
            # step kernel still samples with the old depth and applies vertical advection to the new one
            z_new = self._mix(el.dev('lon', torch.float64), el.dev('lat', torch.float64), z, el.positions_f32)
        elif self._tv_nonzero:
            # no mixing: the buoyancy move (oceandrift.py:201-205), after the moves of this step have read the start-of-step depth
            # and before vertical advection, which the step kernel applies to this new buffer
            z_new = self._buoyancy(z)
        elif stokes_inp is not None and wgrp is not None:
            # update() moves with the Stokes drift BEFORE vertical advection (oceandrift.py:196-205): the Stokes profile
            # must see the start-of-step depth, so vertical advection writes into a copy that replaces z afterwards
            z_new = z.clone()
        # the random-walk draws come last, after the mixing loop's (update() runs before horizontal_diffusion(),
        # basemodel/__init__.py:2272-2280): the legacy generator is shared, so the order of the calls is part of the result
        rand = None
        if D != 0 and not split_diffusion:
            rand = tuple(self._device_normals(n, 2, salt=1))
        eng.step_oceandrift(g, self.get_config('drift:advection_scheme'), t, self.time_step,
                            el.dev('lon', torch.float64), el.dev('lat', torch.float64), z, factor=fac, moving=moving,
                            truncate_below=self.get_config('drift:truncate_ocean_model_below_m'),
                            wind=wind, wdf=el.dev('wind_drift_factor'),
                            wind_drift_depth=self.get_config('drift:wind_drift_depth'), w_group=wgrp,
                            w_at_surface=self.get_config('drift:vertical_advection_at_surface'), rand=rand,
                            diffusivity=float(D), pos_f32=el.positions_f32, z_update=z_new,
                            noise=d_ncur, noise_kinds=nkinds, wind_noise=d_nwind, chain=chain)
        if stokes_inp is not None:
            self.stokes_drift(_inputs=stokes_inp)
        if z_new is not None:
            el.set_dev('z', z_new)
        el.positions_f32 = False
        if split_diffusion:
            OpenDriftSimulation.horizontal_diffusion(self)
        return True

    def update_and_diffuse(self):
        """One time step: fused kernel when the stock recipe applies, else the helpers one by one."""
        if self._fused_ok() and self._step_fused():
            return
        _ = self.environment          # start-of-step environment, before anything moves
        if self.get_config('drift:vertical_mixing'):
            t64 = self.engine.torch.float64
            self._start_positions = (self.elements.dev('lon', t64).clone(), self.elements.dev('lat', t64).clone(),
                                     self.elements.positions_f32)
        self.update()
        OpenDriftSimulation.horizontal_diffusion(self)
