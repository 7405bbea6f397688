"""SedimentDrift on the GPU hot path: the reference's sediment model (opendrift/models/sedimentdrift.py) with the same element type,
required variables, configuration key and update() recipe:

    update():  advect_ocean_current -> vertical_advection -> advect_wind -> stokes_drift -> vertical_mixing -> resuspension

Settling (bottom_interaction, :108-116) runs inside the fused mixing loop (od_vertical_mixing_settle, one launch per step) and
resuspension (:118-126) is one elementwise launch (od_resuspend).  The reference decides in every inner iteration, over the whole
element array, whether bottom_interaction is called at all (some element below Zmin before the lift).  An element that cannot
decide that alone -- it ends an iteration exactly at Zmin, still moving, without having been below -- makes the step's mixing run
again on the per-iteration path with the Python bottom_interaction, from the same draws.
"""
import numpy as np

from ..config import CONFIG_LEVEL_ESSENTIAL
from .oceandrift import OceanDrift, Lagrangian3DArray


class SedimentElement(Lagrangian3DArray):
    """sedimentdrift.py:28-36"""
    variables = Lagrangian3DArray.add_variables([
        ('settled', {'dtype': np.uint8, 'units': '1', 'default': 0}),        # 0 is active, 1 is settled (never written)
        ('terminal_velocity', {'dtype': np.float32, 'units': 'm/s', 'default': -0.001})])


class SedimentDrift(OceanDrift):
    """Model for sediment drift (sedimentdrift.py:39-126)."""
    ElementType = SedimentElement
    # general:coastline_action stays 'none' here; the reference's default for this model is 'previous' (against the GSHHG mask)
    _coast_reference_default = ('previous', 'move elements that reach that mask back to their previous positions')
    # the settling decision of the reference is taken over the whole element array; a shard sees only its own elements
    _distributed_refusal = 'SedimentDrift'

    # sedimentdrift.py:44-60
    required_variables = {
        'x_sea_water_velocity': {'fallback': 0},
        'y_sea_water_velocity': {'fallback': 0},
        'sea_surface_height': {'fallback': 0},
        'upward_sea_water_velocity': {'fallback': 0},
        'x_wind': {'fallback': 0},
        'y_wind': {'fallback': 0},
        'sea_surface_wave_stokes_drift_x_velocity': {'fallback': 0},
        'sea_surface_wave_stokes_drift_y_velocity': {'fallback': 0},
        'sea_surface_wave_period_at_variance_spectral_density_maximum': {'fallback': 0},
        'sea_surface_wave_mean_period_from_variance_spectral_density_second_frequency_moment': {'fallback': 0},
        'land_binary_mask': {'fallback': None},
        'ocean_vertical_diffusivity': {'fallback': 0.02, 'profiles': True},
        'ocean_mixed_layer_thickness': {'fallback': 50},
        'sea_floor_depth_below_sea_level': {'fallback': 10000},
    }

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._add_config({
            'vertical_mixing:resuspension_threshold': {'type': 'float', 'default': 0.2, 'min': 0, 'max': 3, 'units': 'm/s',
                                                       'description': 'Sedimented particles will be resuspended if bottom current '
                                                                      'shear exceeds this value.',
                                                       'level': CONFIG_LEVEL_ESSENTIAL}})
        self._set_config_default('drift:vertical_mixing', True)

    def update(self):
        """sedimentdrift.py:82-104"""
        self.advect_ocean_current()
        self.vertical_advection()
        self.advect_wind()
        self.stokes_drift()
        self.vertical_mixing()
        self.resuspension()

    def bottom_interaction(self, seafloor_depth):
        """sedimentdrift.py:106-116: elements at or below the sea floor settle (moving = 0).  Called from the per-iteration mixing
        path; the settling launch does the same on the device."""
        settling = np.logical_and(self.elements.z <= seafloor_depth, self.elements.moving == 1)
        if np.sum(settling) > 0:
            self.elements.moving[settling] = 0

    def resuspension(self):
        """sedimentdrift.py:118-126 on the device (od_resuspend): settled elements where the step's current is faster than
        vertical_mixing:resuspension_threshold move again, 1 cm higher."""
        eng, el, torch = self.engine, self.elements, self.engine.torch
        if len(el) == 0:
            return
        env = self.environment
        el.set_dev('z', self._z_for_sampling())
        eng.resuspend(env.dev('x_sea_water_velocity', eng), env.dev('y_sea_water_velocity', eng),
                      self.get_config('vertical_mixing:resuspension_threshold'), el.dev('moving', torch.int32), el.dev('z'))

    def _overridden_mixing_hooks(self):
        """SedimentDrift's own bottom_interaction is served inside the settling launch.  A subclass that overrides any hook gets the
        per-iteration path, with bottom_interaction (its own or SedimentDrift's) called from Python."""
        hooks = super()._overridden_mixing_hooks()
        if hooks == ['bottom_interaction'] and type(self).bottom_interaction is SedimentDrift.bottom_interaction:
            return []
        return hooks

    def _mix(self, lon0, lat0, z_in, pos_f32):
        if self._overridden_mixing_hooks():
            return super()._mix(lon0, lat0, z_in, pos_f32)
        eng, el = self.engine, self.elements
        m = self._mix_setup(lon0, lat0, z_in, pos_f32)
        rows = self._mix_draws(m)
        z_out, moving, status, undecided = eng.vertical_mixing_settle(
            m['g'], self.time, lon0, lat0, z_in, m['dt_mix'], m['ntimes'], terminal_velocity=m['tv'], rand=rows,
            seafloor_action=m['action'], status=m['status'], seafloor_code=m['code'], **m['common'])
        if undecided:
            # the launch left z, moving and status as they were: the step again, deciding 'below' over all elements
            return self._mix_iterations(m, ['bottom_interaction'], rows=rows)
        el.set_dev('moving', moving)
        if status is not None:
            el.set_dev('status', status)
        if m['action'] == 2 and eng.last_mix_deactivated:
            self._seafloor_deactivated()
        return z_out
