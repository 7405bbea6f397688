"""PhysicsMethods mixin -- the advection helpers model subclasses call from update(), with the
reference's signatures (opendrift/models/physics_methods.py): advect_ocean_current(factor=1) :611-691,
advect_wind(factor=1) :712-791.  Each call is one kernel launch on the device-resident elements; the
start-of-step environment is the one sampled by the run loop (self.environment)."""
import numpy as np


def seawater_dynamic_viscosity(T, S, model='sharqawy'):
    """Dynamic viscosity of sea water in Pa s (:139-178), NumPy on host arrays: Sharqawy et al. (2010) for T in degrees Celsius
    and S in g/kg, or with model='ladim' the linear fit of the LADIM code."""
    if model == 'ladim':
        return 0.001 * (1.7915 - 0.0538 * T + 0.0007 * (T ** (2.0)) + 0.0023 * S)
    if model != 'sharqawy':
        raise ValueError(f'Model {model} not available')
    mu_pure = 4.2844e-5 + 1.0 / (0.157 * (T + 64.993) ** 2 - 91.296)
    a = 1.541 + 1.998e-2 * T - 9.52e-5 * T ** 2
    b = 7.974 - 7.561e-2 * T + 4.724e-4 * T ** 2
    return mu_pure * (1 + a * (S / 1000) + b * (S / 1000) ** 2)


class PhysicsMethods:

    @staticmethod
    def sea_water_density(T=10., S=35.):
        """Density of sea water at one atmosphere (:574-609; Fofonoff and Millard 1983, UNESCO technical papers in marine science
        44), NumPy on host arrays: T in degrees Celsius, S in PSU.  Raises ValueError when the largest T exceeds 100."""
        if np.atleast_1d(T).max() > 100:
            raise ValueError('Temperature should be in celcius, but is > 100')
        # pure water (Bigg 1967), then the salinity terms
        r1 = ((((6.536332E-09 * T - 1.120083E-06) * T + 1.001685E-04) * T - 9.095290E-03) * T + 6.793952E-02) * T - 28.263737
        r2 = (((5.3875E-09 * T - 8.2467E-07) * T + 7.6438E-05) * T - 4.0899E-03) * T + 8.24493E-01
        r3 = (-1.6546E-06 * T + 1.0227E-04) * T - 5.72466E-03
        sigma = r1 + (4.8314E-04 * S + r3 * np.sqrt(S) + r2) * S
        return sigma + 28.106331 + 1000.

    def _current_group(self, t):
        # the first reader that covers any stage time of the step that starts at t (a reader whose coverage begins inside
        # the step serves the later stages; the stages before it get the fallback, as in the reference)
        rx = self._current_readers(t)[0]
        r = rx[0] if rx else None
        if r is None or not hasattr(r, 'group_of'):
            return None
        if 'y_sea_water_velocity' not in r.variables:
            return None                              # the components come from different sources: staged recipe
        g, c = r.group_of('x_sea_water_velocity')
        g2, c2 = r.group_of('y_sea_water_velocity')
        assert g is g2 and (c, c2) == (0, 1), 'current components must come from one reader'
        return g

    def _stage_times(self, t):
        """Times at which advect_ocean_current samples the current (:611-691)."""
        scheme, dt = self.get_config('drift:advection_scheme'), self.time_step
        return [t] if scheme == 'euler' else ([t, t + dt / 2] if scheme == 'runge-kutta' else [t, t + dt / 2, t + dt])

    def _current_readers(self, t):
        ts = self._stage_times(t)
        return (self.env.readers_for_times('x_sea_water_velocity', ts), self.env.readers_for_times('y_sea_water_velocity', ts))

    def _current_chain(self, t):
        """[primary group, further groups ...] when the current's reader priority list can run inside the step kernels: every
        reader of the list is gridded, serves both components as one two-component group, and the list is short enough
        (include/odcuda.h: OD_MAX_CHAIN further groups).  None otherwise (staged recipe)."""
        from .. import _lib
        rx, ry = self._current_readers(t)
        if len(rx) < 2 or len(rx) != len(ry) or any(a is not b for a, b in zip(rx, ry)) or len(rx) > 1 + _lib.OD_MAX_CHAIN:
            return None
        if any(hasattr(r, 'has_ensembles') and r.has_ensembles() for r in rx):
            return None
        groups = []
        for r in rx:
            if not hasattr(r, 'group_of'):
                return None
            g, c = r.group_of('x_sea_water_velocity')
            g2, c2 = r.group_of('y_sea_water_velocity')
            if g is not g2 or (c, c2) != (0, 1):
                return None
            groups.append(g)
        return groups

    def _current_needs_reader_loop(self, t):
        """True when the current cannot be sampled from ONE two-component field group: several readers in priority order,
        or x and y components from different readers (the reference resolves every variable on its own, environment.py:613-780)."""
        rx, ry = self._current_readers(t)
        if len(rx) > 1 or len(ry) > 1:
            return True
        if any(getattr(r, 'host_callback', False) for r in rx + ry):
            return True                  # values computed on the host (readers/continuous.py): stage by stage through device_sample()
        if any(hasattr(r, 'has_ensembles') and r.has_ensembles('x_sea_water_velocity') for r in rx):
            return True                  # ensemble blocks: the member of an element depends on which elements a call serves (staged recipe)
        return len(rx) + len(ry) > 0 and (len(rx) != len(ry) or rx[0] is not ry[0])

    def _device_factor(self, factor, name):
        """factor * elements.<name> with NumPy's dtype rules (int/float scalar factors are weak)."""
        eng, torch = self.engine, self.engine.torch
        p = self.elements.dev(name)
        if isinstance(factor, (int, float)) and factor == 1:
            return p
        if isinstance(factor, (int, float)):
            return p * p.new_tensor(factor)
        f = factor if isinstance(factor, torch.Tensor) else eng.to_device(np.ascontiguousarray(factor))
        return f * p

    def advect_ocean_current(self, factor=1):
        eng, el, torch = self.engine, self.elements, self.engine.torch
        scheme = self.get_config('drift:advection_scheme')
        fac = self._device_factor(factor, 'current_drift_factor') if 'current_drift_factor' in el.variables else None
        if fac is not None and fac.dtype not in (torch.float32, torch.float64):
            fac = fac.to(torch.float64)
        moving = el.dev('moving')
        if moving.dtype != torch.int32:
            moving = moving.to(torch.int32)
        lon, lat = el.dev('lon', torch.float64), el.dev('lat', torch.float64)
        g = self._current_group(self.time)
        trunc = self.get_config('drift:truncate_ocean_model_below_m', None)
        ra = self.env.reader_for('x_sea_water_velocity', self.time)
        chain = ()
        if self._current_needs_reader_loop(self.time):
            # several current readers in priority order (e.g. a nested model inside a coarser one): every stage needs the
            # reference's reader loop on the still-missing elements -- inside the kernel when the list is made of gridded
            # two-component groups (reader chain), else stage by stage
            groups = self._current_chain(self.time)
            if groups is None:
                return self._advect_ocean_current_staged(scheme, fac, moving, lon, lat)
            g, chain = groups[0], tuple(groups[1:])
        if g is None and ra is not None and hasattr(ra, 'analytic_desc'):
            # analytical reader on a projected plane: the stage loop samples it on the device (od_analytic_advect)
            if any(x > 0 for x in self._uncertainty()[:2]):
                raise NotImplementedError('drift:current_uncertainty with an analytical reader is not on the GPU path')
            k1 = None
            view = getattr(self, '_env_view', None)
            if view is not None and 'x_sea_water_velocity' in view:
                k1 = (view.dev('x_sea_water_velocity', eng), view.dev('y_sea_water_velocity', eng))
            t, dt = self.time, self.time_step
            eng.analytic_advect(ra.analytic_desc(), scheme, (ra.seconds(t), ra.seconds(t + dt / 2), ra.seconds(t + dt)),
                                dt.total_seconds(), lon, lat, factor=fac, moving=moving, k1=k1, pos_f32=el.positions_f32)
            el.positions_f32 = False
            return
        if g is None:
            # no gridded current reader: constant / fallback current -> plain update_positions (Euler == RK)
            env = self.environment
            u, v = env.dev('x_sea_water_velocity', eng), env.dev('y_sea_water_velocity', eng)
            if fac is None:
                self.update_positions(u, v)
            else:
                self.update_positions(fac * u if fac.dtype == u.dtype else fac.to(torch.float64) * u.to(torch.float64),
                                      fac * v if fac.dtype == v.dtype else fac.to(torch.float64) * v.to(torch.float64))
            return
        # k1 is the start-of-step environment if somebody already materialised it (e.g. a subclass modified it)
        k1 = None
        view = getattr(self, '_env_view', None)
        if view is not None and 'x_sea_water_velocity' in view:
            k1 = (view.dev('x_sea_water_velocity', eng), view.dev('y_sea_water_velocity', eng))
        noise, kinds = None, 0
        cu, cuu, _ = self._uncertainty()
        if cu > 0 or cuu > 0:
            from ..engine import draw_uncertainty
            if k1 is None:                    # the step's environment has not been drawn yet: stage 0 included
                arr, kinds, _ = draw_uncertainty(lon.numel(), scheme, cu, cuu, stage0=getattr(self, '_noise0', None))
            else:                             # stages 2..4 only (the step's environment already carries its draws)
                sub = {'euler': None, 'runge-kutta': 'euler', 'runge-kutta4': 'runge-kutta4'}[scheme]
                arr = None
                if sub is not None:
                    nst = 1 if scheme == 'runge-kutta' else 3
                    arr = np.zeros((4, 2, 2, lon.numel()))
                    kinds = (1 if cu > 0 else 0) | (2 if cuu > 0 else 0)
                    for st in range(1, 1 + nst):
                        if cu > 0:
                            arr[st, 0, 0] = np.random.normal(0, cu, lon.numel())
                            arr[st, 0, 1] = np.random.normal(0, cu, lon.numel())
                        if cuu > 0:
                            arr[st, 1, 0] = np.random.uniform(-cuu, cuu, lon.numel())
                            arr[st, 1, 1] = np.random.uniform(-cuu, cuu, lon.numel())
            noise = eng.to_device(arr) if arr is not None else None
        eng.advect_current(g, scheme, self.time, self.time_step, lon, lat,
                           self._z_for_sampling() if g.desc.nz > 1 else None, factor=fac, moving=moving, k1=k1,
                           truncate_below=trunc, pos_f32=el.positions_f32, noise=noise, noise_kinds=kinds if noise is not None else 0,
                           chain=chain)
        el.positions_f32 = False

    def _advect_ocean_current_staged(self, scheme, fac, moving, lon, lat):
        """advect_ocean_current (:611-691) stage by stage for a current that comes from several readers: each stage
        velocity is a full Environment.device_environment call (reader priority loop, fallback), mid-points and the final
        move are geodesic launches.  Slower than the fused kernels (8 launches per RK4 step instead of 1); only used when
        more than one reader provides the current."""
        eng, el, torch = self.engine, self.elements, self.engine.torch
        uv = ['x_sea_water_velocity', 'y_sea_water_velocity']
        env = self.environment                       # start-of-step environment (with its uncertainty draws)
        k1u, k1v = env.dev(uv[0], eng), env.dev(uv[1], eng)
        t, dt = self.time, self.time_step
        dts = np.float32(dt.total_seconds())
        z = self._z_truncated()

        def stage(ku, kv, when):
            # x0 (+) 0.5 dt k with the reference's float32 azimuth / speed / distance (:629-635)
            az = torch.rad2deg(torch.atan2(ku, kv))
            dist = torch.sqrt(ku * ku + kv * kv) * dts * np.float32(0.5)
            mlon, mlat = lon.clone(), lat.clone()
            eng.geod_fwd(mlon, mlat, az.to(torch.float64), dist.to(torch.float64))
            d_env, _ = self.env.device_environment(uv, when, mlon, mlat, z, pos_f32=False)
            self._add_uncertainty(d_env)
            return d_env[uv[0]], d_env[uv[1]]

        if scheme == 'euler':
            ru, rv = k1u, k1v
        else:
            k2u, k2v = stage(k1u, k1v, t + dt / 2)
            if scheme == 'runge-kutta':
                ru, rv = k2u, k2v
            else:
                k3u, k3v = stage(k2u, k2v, t + dt / 2)
                k4u, k4v = stage(k3u, k3v, t + dt)                       # half step, end time (:660-670)
                ru = (k1u + 2 * k2u + 2 * k3u + k4u) / 6.0
                rv = (k1v + 2 * k2v + 2 * k3v + k4v) / 6.0
        if fac is None:
            self.update_positions(ru, rv)
        elif fac.dtype == ru.dtype:
            self.update_positions(ru * fac, rv * fac)
        else:
            self.update_positions(ru.to(torch.float64) * fac.to(torch.float64), rv.to(torch.float64) * fac.to(torch.float64))

    # -- small helpers model subclasses call from update() (physics_methods.py:885-891, basemodel/__init__.py:4524-4529) -----------
    def wind_speed(self):
        return np.sqrt(self.environment.x_wind**2 + self.environment.y_wind**2)

    def current_speed(self):
        return np.sqrt(self.environment.x_sea_water_velocity**2 + self.environment.y_sea_water_velocity**2)

    def simulation_direction(self):
        """1 for a forward simulation, -1 for a backward simulation"""
        return -1 if self.time_step.days < 0 else 1

    def advect_with_sea_ice(self, factor=1):
        """physics_methods.py:693-710: drift with the sea ice -- its velocity from a reader, else Nordam's rule of thumb
        (current + 1.5 % of the wind) -- times `factor` (OpenOil: the ice coverage factor k_ice, a float32 array)."""
        eng, torch = self.engine, self.engine.torch
        env = self.environment
        if 'sea_ice_x_velocity' in env:
            u, v = env.dev('sea_ice_x_velocity', eng), env.dev('sea_ice_y_velocity', eng)
        else:
            if 'x_sea_water_velocity' not in env:
                return
            u, v = env.dev('x_sea_water_velocity', eng), env.dev('y_sea_water_velocity', eng)
            if 'x_wind' in env:
                # float32 + (Python float * float32): float32 arithmetic
                c = u.new_tensor(0.015)
                u, v = u + c * env.dev('x_wind', eng), v + c * env.dev('y_wind', eng)
        if isinstance(factor, (int, float)):
            if factor != 1:
                f = u.new_tensor(factor)                  # weak scalar: the products stay float32
                u, v = f * u, f * v
        else:
            f = factor if isinstance(factor, torch.Tensor) else eng.to_device(np.ascontiguousarray(factor))
            if f.dtype != u.dtype:                        # NumPy's promotion
                rt = torch.promote_types(f.dtype, u.dtype)
                f, u, v = f.to(rt), u.to(rt), v.to(rt)
            u, v = f * u, f * v
        self.update_positions(u, v)

    def advect_wind(self, factor=1):
        """Wind drift of elements near the surface (:712-791): wind_drift_factor, linearly reduced to zero at
        drift:wind_drift_depth; relative_wind optional."""
        eng, el, torch = self.engine, self.elements, self.engine.torch
        env = self.environment
        if 'x_wind' not in env:
            return
        xw, yw = env.dev('x_wind', eng), env.dev('y_wind', eng)
        wdf = el.dev('wind_drift_factor')
        z = el.dev('z')
        wdd = self.get_config('drift:wind_drift_depth', 0) or 0
        surface = z >= -abs(wdd)
        if wdd != 0:
            wdd_t = torch.full_like(z, abs(wdd), dtype=torch.float64)
            w = wdf.to(torch.float64) * (wdd_t + z.to(torch.float64)) / wdd_t
            w = torch.where(z > 0, wdf.to(torch.float64), w)
        else:
            w = wdf.clone()
        w = torch.where(surface, w, torch.zeros_like(w))
        if self.get_config('drift:relative_wind', False):
            xw = xw - env.dev('x_sea_water_velocity', eng)
            yw = yw - env.dev('y_sea_water_velocity', eng)
        if isinstance(factor, (int, float)) and factor == 1:
            xv, yv = xw.to(w.dtype) * w, yw.to(w.dtype) * w
        else:
            f = factor if isinstance(factor, torch.Tensor) else (
                eng.to_device(np.ascontiguousarray(factor)) if not isinstance(factor, (int, float)) else factor)
            xv, yv = xw.to(w.dtype) * w * f, yw.to(w.dtype) * w * f
        self.update_positions(xv, yv)

    def _stokes_inputs(self):
        """Start-of-step samples the Stokes move needs (device float32 tensors) + the reference's collective
        decisions (:799-812, :893-906).  Returns None when the reference would return early."""
        eng = self.engine
        sx, sy = 'sea_surface_wave_stokes_drift_x_velocity', 'sea_surface_wave_stokes_drift_y_velocity'
        wanted = [sx, sy, 'sea_surface_wave_significant_height', 'x_wind', 'y_wind']
        if getattr(self, '_env_view', None) is not None or any(x > 0 for x in self._uncertainty()):
            env = self.environment            # already materialised (helper recipes), or it must carry its uncertainty draws
        else:
            # the fused step never materialises the whole start-of-step environment: sample only what the Stokes move reads
            el, torch = self.elements, self.engine.torch
            names = [v for v in wanted if v in self._env_variables]
            d_env, _ = self.env.device_environment(names, self.time, el.dev('lon', torch.float64), el.dev('lat', torch.float64),
                                                   self._z_truncated(), pos_f32=el.positions_f32)
            from .basemodel import EnvironmentView
            env = EnvironmentView(d_env)
        us, vs = env.dev(sx, eng), env.dev(sy, eng)
        if eng.minmax(us, vs)[1] == 0:
            return None                                   # 'No Stokes drift velocity available'
        hs = env.dev('sea_surface_wave_significant_height', eng) if 'sea_surface_wave_significant_height' in env else None
        xw = env.dev('x_wind', eng) if 'x_wind' in env else None
        yw = env.dev('y_wind', eng) if 'y_wind' in env else None
        if hs is not None and eng.minmax(hs)[1] > 0:
            mode = 0
        else:
            any_wind = False
            for w in (xw, yw):
                if w is not None:
                    lo, hi = eng.minmax(w)
                    any_wind |= (hi > 0 or lo < 0)
            mode = 1 if any_wind else 2
        return us, vs, hs, xw, yw, mode

    def _windsea_swell_arrays(self, profile):
        """The six float32 tensors of the swell / wind-sea partition of the wave field (:418-455) for the windsea_swell profile,
        else None; the model must have declared these variables."""
        if profile != 'windsea_swell':
            return None
        env = self.environment
        names = ('sea_surface_swell_wave_to_direction', 'sea_surface_swell_wave_peak_period_from_variance_spectral_density',
                 'sea_surface_swell_wave_significant_height', 'sea_surface_wind_wave_to_direction',
                 'sea_surface_wind_wave_mean_period', 'sea_surface_wind_wave_significant_height')
        missing = [v for v in names if v not in env]
        if missing:
            raise AttributeError('the windsea_swell Stokes profile needs the environment variables %s '
                                 '(add them to required_variables)' % missing)
        return tuple(env.dev(v, self.engine) for v in names)

    def stokes_drift(self, factor=1, _inputs='sample'):
        """Stokes drift with a depth profile (:793-848): monochromatic / exponential / Phillips (:332-416)."""
        if not self.get_config('drift:stokes_drift', False):
            return
        profile = self.get_config('drift:stokes_drift_profile', default='monochromatic')
        inp = self._stokes_inputs() if _inputs == 'sample' else _inputs
        if inp is None:
            return
        us, vs, hs, xw, yw, mode = inp
        eng, el, torch = self.engine, self.elements, self.engine.torch
        ww = self._windsea_swell_arrays(profile)
        if not isinstance(factor, (int, float)):
            factor = factor if isinstance(factor, torch.Tensor) else eng.to_device(np.ascontiguousarray(factor))
            if factor.dtype not in (torch.float32, torch.float64):
                factor = factor.to(torch.float64)
        moving = el.dev('moving')
        if moving.dtype != torch.int32:
            moving = moving.to(torch.int32)
        eng.stokes_drift(el.dev('lon', torch.float64), el.dev('lat', torch.float64), self._z_for_sampling(), us, vs, hs,
                         xw, yw, moving, self.time_step.total_seconds(), mode, profile, factor=factor, windsea_swell=ww)
        el.positions_f32 = False
