"""PlastDrift (plastics) on the GPU path: the reference's model class (opendrift/models/plastdrift.py) with the same element type
(PlastElement :23-29), required variables (:44-57), configuration (:60-78) and update() (:80-107):

    update():  advect_ocean_current -> update_particle_depth -> stokes_drift -> advect_wind

update_particle_depth draws a new depth for every active element with vertical_mixing:mixingmodel = 'analytical' (the default),
z = -np.random.exponential(scale=K / terminal_velocity), or runs the random-walk mixing loop with 'randomwalk'.  After the current
move, the rest of update() is ONE launch per step (od_plast_step, csrc/od_plast.cuh): the new depth, the Stokes move and the wind move
at that depth.  With 'randomwalk' the mixing launch comes first and od_plast_step does the two moves.  The Stokes decisions the
reference takes over the whole element array come from reductions on the device before the launch (_stokes_inputs).
"""
import numpy as np

from ..config import CONFIG_LEVEL_ESSENTIAL, CONFIG_LEVEL_ADVANCED
from .oceandrift import OceanDrift, Lagrangian3DArray
from .physics_methods import PhysicsMethods


class PlastElement(Lagrangian3DArray):
    """plastdrift.py:23-29"""
    variables = Lagrangian3DArray.add_variables([
        ('terminal_velocity', {'dtype': np.float32, 'units': 'm/s', 'level': CONFIG_LEVEL_ESSENTIAL,
                               'description': 'Positive value means rising particles (positive buoyancy)', 'default': 0.01})])


class PlastDrift(OceanDrift):
    """Plastics drifting with the ocean current, Stokes drift and wind drag (plastdrift.py:32-107)."""
    ElementType = PlastElement
    # general:coastline_action stays 'none' here; the reference's default for this model is 'previous' (against the GSHHG mask)
    _coast_reference_default = ('previous', 'move elements that reach that mask back to their previous positions')
    # the Stokes decisions and the legacy generator's draws are taken over the whole element array; a shard sees only its own
    _distributed_refusal = 'PlastDrift'

    # plastdrift.py:44-57
    required_variables = {
        'x_sea_water_velocity': {'fallback': 0},
        'y_sea_water_velocity': {'fallback': 0},
        'sea_surface_height': {'fallback': 0},
        'sea_surface_wave_stokes_drift_x_velocity': {'fallback': 0},
        'sea_surface_wave_stokes_drift_y_velocity': {'fallback': 0},
        'sea_surface_wave_significant_height': {'fallback': 0},
        'x_wind': {'fallback': 0},
        'y_wind': {'fallback': 0},
        'ocean_vertical_diffusivity': {'fallback': 0.02, 'profiles': True},
        'ocean_mixed_layer_thickness': {'fallback': 50},
        'sea_floor_depth_below_sea_level': {'fallback': 10000},
        'land_binary_mask': {'fallback': None},
    }

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._add_config({
            'vertical_mixing:mixingmodel': {'type': 'enum', 'enum': ['randomwalk', 'analytical'], 'default': 'analytical',
                                            'level': CONFIG_LEVEL_ADVANCED,
                                            'description': 'Scheme to be used for vertical turbulent mixing'}})
        self._set_config_default('drift:vertical_mixing', True)
        self._set_config_default('drift:vertical_advection', True)
        self._set_config_default('drift:use_tabularised_stokes_drift', True)
        self._set_config_default('vertical_mixing:diffusivitymodel', 'windspeed_Sundby1983')

    def update(self):
        """plastdrift.py:80-92.  The reference's update() does not call vertical_advection(), although its default is True."""
        self.advect_ocean_current()
        t = type(self)
        if (t.update_particle_depth is PlastDrift.update_particle_depth and t.stokes_drift is PhysicsMethods.stokes_drift
                and t.advect_wind is PhysicsMethods.advect_wind and not self.get_config('drift:relative_wind')):
            self._after_current()
            return
        self.update_particle_depth()
        self.stokes_drift()
        self.advect_wind()

    def update_particle_depth(self):
        """plastdrift.py:94-107: the random-walk mixing loop, or a depth drawn from an exponential distribution whose scale is
        K / terminal_velocity (one launch, od_plast_step; the sea floor is left to the next step's interact_with_seafloor)."""
        if self.get_config('drift:vertical_mixing') is not True:
            return
        model = self.get_config('vertical_mixing:mixingmodel')
        if model == 'randomwalk':
            self.vertical_mixing()
        elif model == 'analytical':
            self._launch(submerge=True, stokes=None, wind=None)

    # -- the device step ------------------------------------------------------------------------------------------------------------
    def _after_current(self):
        """update_particle_depth -> stokes_drift -> advect_wind: the mixing launch first with 'randomwalk', then one od_plast_step."""
        mixing = self.get_config('drift:vertical_mixing') is True
        model = self.get_config('vertical_mixing:mixingmodel')
        if mixing and model == 'randomwalk':
            self.vertical_mixing()
        stokes = None
        if self.get_config('drift:stokes_drift', False):
            inp = self._stokes_inputs()
            if inp is not None:
                profile = self.get_config('drift:stokes_drift_profile', default='monochromatic')
                stokes = tuple(inp) + (profile, self._windsea_swell_arrays(profile))
        env = self.environment
        wind = None
        if 'x_wind' in env:
            wind = (self._env_f32('x_wind'), self._env_f32('y_wind'), self.get_config('drift:wind_drift_depth', 0) or 0)
        self._launch(submerge=mixing and model == 'analytical', stokes=stokes, wind=wind)

    def _launch(self, submerge, stokes, wind):
        eng, el, torch = self.engine, self.elements, self.engine.torch
        n = len(el)
        if n == 0 or (not submerge and stokes is None and wind is None):
            return
        z = self._z_for_sampling()
        sub = None
        if submerge:
            tv = el.dev('terminal_velocity')
            if tv.dtype not in (torch.float32, torch.float64):
                tv = el.dev('terminal_velocity', torch.float64)
            draws = None
            if self.get_config('gpu:rng') == 'numpy':
                # np.random.exponential(scale, size=n) of the legacy generator is scale * standard_exponential(n), draw by draw
                draws = eng.to_device(np.random.standard_exponential(n))
            ids = el.dev('ID')
            if ids.dtype != torch.int32:
                ids = ids.to(torch.int32)
            sub = (self._env_f32('ocean_vertical_diffusivity'), tv.contiguous(), draws, ids, getattr(self, '_seed', 0),
                   self.steps_calculation)
        wnd = None
        if wind is not None:
            wdf = el.dev('wind_drift_factor')
            if wdf.dtype not in (torch.float32, torch.float64):
                wdf = el.dev('wind_drift_factor', torch.float64)
            wnd = (wind[0], wind[1], wdf.contiguous(), wind[2])
        moving = el.dev('moving')
        if moving.dtype != torch.int32:
            moving = moving.to(torch.int32)
        z_new = eng.plast_step(el.dev('lon', torch.float64), el.dev('lat', torch.float64), moving, z,
                               self.time_step.total_seconds(), submerge=sub, stokes=stokes, wind=wnd)
        if stokes is not None or wind is not None:
            el.positions_f32 = False
        if z_new is not None:
            el.set_dev('z', z_new)
