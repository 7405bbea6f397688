"""LarvalFish (fish eggs and larvae) on the GPU path: the reference's model class (opendrift/models/larvalfish.py) with the same element
type (LarvalFishElement :26-55), required variables (:69-84), configuration (:87-102) and update() (:255-265):

    update():  update_fish_larvae -> advect_ocean_current -> stokes_drift -> update_terminal_velocity -> vertical_mixing
               -> larvae_vertical_migration

Eggs develop with the temperature and hatch into larvae, which grow (Folkvord 2005) and swim down before 12:00 UTC and up after it.
Every element has Sundby's (1983) egg buoyancy as its terminal velocity in the mixing loop.  Without vertical_mixing:TSprofiles
(refused here) that velocity depends on the start-of-step temperature and salinity and on diameter and neutral_buoyancy_salinity
only, so the value the reference recomputes at every inner iteration is one value per element and step.  A step is therefore
od_larval_develop (hatching, growth, length and the terminal velocity; csrc/od_larval.cuh) before the current move, the current and
Stokes launches, ONE fused mixing launch, and od_larval_migrate.  A subclass that overrides update_fish_larvae, fish_growth,
larvae_vertical_migration or update_terminal_velocity takes the helpers one by one; one that overrides update_terminal_velocity
also takes the per-iteration mixing path.
"""
import numpy as np

from ..config import CONFIG_LEVEL_ADVANCED
from .oceandrift import OceanDrift, Lagrangian3DArray


class LarvalFishElement(Lagrangian3DArray):
    """larvalfish.py:26-55"""
    variables = Lagrangian3DArray.add_variables([
        ('diameter', {'dtype': np.float32, 'units': 'm', 'default': 0.0014}),
        ('neutral_buoyancy_salinity', {'dtype': np.float32, 'units': 'PSU', 'default': 31.25}),
        ('stage_fraction', {'dtype': np.float32, 'units': '', 'default': 0.}),
        ('hatched', {'dtype': np.uint8, 'units': '', 'default': 0}),
        ('length', {'dtype': np.float32, 'units': 'mm', 'default': 0}),
        ('weight', {'dtype': np.float32, 'units': 'mg', 'default': 0.08}),
        ('survival', {'dtype': np.float32, 'units': '', 'default': 1.})])


class LarvalFish(OceanDrift):
    """Fish eggs that hatch into larvae, which grow and migrate vertically by day and night (larvalfish.py:58-265)."""
    ElementType = LarvalFishElement
    # the temperature check and the legacy generator's mixing draws are taken over the whole element array; a shard sees its own
    _distributed_refusal = 'LarvalFish'

    # larvalfish.py:69-84
    required_variables = {
        'x_sea_water_velocity': {'fallback': 0},
        'y_sea_water_velocity': {'fallback': 0},
        'sea_surface_height': {'fallback': 0},
        'sea_surface_wave_significant_height': {'fallback': 0},
        'x_wind': {'fallback': 0},
        'y_wind': {'fallback': 0},
        'land_binary_mask': {'fallback': None},
        'sea_floor_depth_below_sea_level': {'fallback': 100},
        'ocean_vertical_diffusivity': {'fallback': 0.01, 'profiles': True},
        'ocean_mixed_layer_thickness': {'fallback': 50},
        'sea_water_temperature': {'fallback': 10, 'profiles': True},
        'sea_water_salinity': {'fallback': 34, 'profiles': True},
        'sea_surface_wave_stokes_drift_x_velocity': {'fallback': 0},
        'sea_surface_wave_stokes_drift_y_velocity': {'fallback': 0},
    }

    # the helpers the fused step stands in for
    _HELPERS = ('update_fish_larvae', 'fish_growth', 'larvae_vertical_migration', 'update_terminal_velocity')

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._add_config({
            'IBM:fraction_of_timestep_swimming': {'type': 'float', 'default': 0.15, 'min': 0.0, 'max': 1.0, 'units': 'fraction',
                                                  'description': 'Fraction of timestep swimming', 'level': CONFIG_LEVEL_ADVANCED}})
        self._set_config_default('drift:vertical_mixing', True)
        self._set_config_default('drift:vertical_mixing_at_surface', True)
        self._set_config_default('drift:vertical_advection_at_surface', True)

    def run(self, *args, **kwargs):
        # An element seeded with hatched outside {0, 1} is neither egg nor larva; when no element is either, the reference's debug
        # message takes the max of an empty array and raises.  Only then does the step need the flags read back for that.
        self._hatched_odd = False
        if hasattr(self, 'elements_scheduled'):
            h = np.atleast_1d(self.elements_scheduled.hatched)
            self._hatched_odd = bool(np.any((h != 0) & (h != 1)))
        return super().run(*args, **kwargs)

    def update(self):
        """larvalfish.py:255-265.  Like the reference, no vertical advection, wind drift or water column stretching."""
        t = type(self)
        fused = all(getattr(t, h) is getattr(LarvalFish, h) for h in self._HELPERS)
        if fused:
            w, hot = self._develop(develop=True, velocity=True)
        else:
            self.update_fish_larvae()
        self.advect_ocean_current()
        self.stokes_drift()
        if fused:
            self._set_terminal_velocity(w, hot)
        else:
            self.update_terminal_velocity()
        self.vertical_mixing()
        self.larvae_vertical_migration()

    # -- the reference's helpers -------------------------------------------------------------------------------------------------
    def update_terminal_velocity(self, Tprofiles=None, Sprofiles=None, z_index=None):
        """larvalfish.py:105-183: Sundby's (1983) terminal velocity of a pelagic egg from the start-of-step temperature and
        salinity, for every element (od_larval_develop with the development switched off)."""
        if Tprofiles is not None or Sprofiles is not None:
            raise NotImplementedError('vertical_mixing:TSprofiles is not on the GPU path')
        w, hot = self._develop(develop=False, velocity=True)
        self._set_terminal_velocity(w, hot)

    def fish_growth(self, weight, temperature):
        """larvalfish.py:185-198: the weight (mg) a larva gains in one time step at a temperature in degrees Celsius, from the
        daily growth rate in percent of Folkvord (2005).  NumPy on host arrays."""
        lw = np.log(weight)
        rate = 1.08 + 1.79 * temperature - 0.074 * temperature * lw - 0.0965 * temperature * lw ** 2 + 0.0112 * temperature * lw ** 3
        g = (np.log(rate / 100. + 1)) * self.time_step.total_seconds() / 86400
        return weight * (np.exp(g) - 1.)

    def update_fish_larvae(self):
        """larvalfish.py:200-231: eggs develop and hatch, larvae grow (od_larval_develop without the terminal velocity).  With a
        fish_growth of a subclass, NumPy on host arrays."""
        if type(self).fish_growth is not LarvalFish.fish_growth:
            self._update_fish_larvae_host()
            return
        self._develop(develop=True, velocity=False)

    def larvae_vertical_migration(self):
        """larvalfish.py:233-253: larvae swim down before 12:00 UTC (the step's start time) and up after it, by
        IBM:fraction_of_timestep_swimming of the distance their swimming speed (Peck et al. 2006) covers in a time step, no higher
        than the surface (od_larval_migrate)."""
        eng, el = self.engine, self.elements
        if len(el) == 0:
            return
        z = self._z_for_sampling().contiguous()
        tens = self._larval_tensors(('hatched', 'length'))
        eng.larval_migrate(tens['hatched'], tens['length'], z, self.get_config('IBM:fraction_of_timestep_swimming'),
                           -1 if self.time.hour < 12 else 1, self.time_step.total_seconds())
        el.set_dev('z', z)

    def _overridden_mixing_hooks(self):
        # LarvalFish's own terminal velocity is constant through the step: the fused mixing launch takes it as it stands
        hooks = super()._overridden_mixing_hooks()
        if type(self).update_terminal_velocity is LarvalFish.update_terminal_velocity:
            hooks.remove('update_terminal_velocity')
        return hooks

    # -- the device step -----------------------------------------------------------------------------------------------------------
    def _larval_tensors(self, names):
        """The element tensors od_larval_* take: hatched uint8 or float64, the others float32 or float64, contiguous."""
        el, torch = self.elements, self.engine.torch
        out = {}
        for v in names:
            t = el.dev(v)
            if t.dtype not in ((torch.uint8, torch.float64) if v == 'hatched' else (torch.float32, torch.float64)):
                t = el.dev(v, torch.float64)
            if not t.is_contiguous():
                t = t.contiguous()
                el.set_dev(v, t)
            out[v] = t
        return out

    def _develop(self, develop, velocity):
        """od_larval_develop.  Returns (the new terminal velocity or None, whether the reference's temperature check raises).
        Raises the reference's zero-size ValueError when no element is an egg or a larva.  The flags are read back only when a
        decision needs them: the temperature comes from a reader, or some seeded hatched lies outside {0, 1}."""
        eng = self.engine
        hot = None
        if velocity:
            c = self._constant_or_none('sea_water_temperature')
            if c is not None:
                hot = bool(np.float32(c) > 100)
        check_staged = develop and getattr(self, '_hatched_odd', True)
        want = (velocity and hot is None) or check_staged
        names = (('hatched', 'stage_fraction', 'weight', 'length') if develop else ()) + \
            (('diameter', 'neutral_buoyancy_salinity') if velocity else ())
        w, flags = eng.larval_develop(self._env_f32('sea_water_temperature'),
                                      self._env_f32('sea_water_salinity') if velocity else None, self._larval_tensors(names),
                                      self.time_step.total_seconds(), develop=develop, velocity=velocity, flags=want)
        if check_staged and not flags & eng.LARVAL_STAGED:
            np.zeros(0, dtype=np.float32).max()      # the max of the (empty) eggs' stage fractions in the reference's debug message
        if velocity and hot is None:
            # sea_water_density: np.max is NaN when some T is, and NaN > 100 is False
            hot = bool(flags & eng.LARVAL_HOT) and not flags & eng.LARVAL_NAN_T
        return w, hot

    def _set_terminal_velocity(self, w, hot):
        if hot:
            raise ValueError('Temperature should be in celcius, but is > 100')
        self.elements.set_dev('terminal_velocity', w)

    def _update_fish_larvae_host(self):
        """update_fish_larvae with a subclass's fish_growth, on host arrays."""
        el, temp = self.elements, self.environment.sea_water_temperature
        eggs = np.where(el.hatched == 0)[0]
        if len(eggs) > 0:
            el.stage_fraction[eggs] += (self.time_step.total_seconds() / 86400) / np.exp(3.65 - 0.145 * temp[eggs])
            hatching = np.where(el.stage_fraction[eggs] >= 1)[0]
            el.hatched[eggs[hatching]] = 1
        larvae = np.where(el.hatched == 1)[0]
        if len(larvae) == 0:
            el.stage_fraction[eggs].max()            # the reference's debug message: raises when there are no eggs either
            return
        el.weight[larvae] += self.fish_growth(el.weight[larvae], temp[larvae])
        w = el.weight[larvae]
        el.length[larvae] = np.exp(2.296 + 0.277 * np.log(w) - 0.005128 * np.log10(w) ** 2)
