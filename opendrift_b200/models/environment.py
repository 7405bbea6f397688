"""Environment: reader registry and get_environment() with the reference's contract
(opendrift/models/basemodel/environment.py:499-923): loop the variable groups over the readers in priority
order on the still-missing particles, cast to float32, apply `environment:constant:*` /
`environment:fallback:*`, return (recarray float32, env_profiles, missing mask).

Two faces:
  * get_environment(...)      NumPy in / NumPy out, for model code and user scripts (host copies);
  * device_environment(...)   device tensors in / device tensors out, used by the step methods.
Both run od_interp for the sampling.  The fused step kernels bypass this class entirely and read the bound
field groups directly; fallback values are baked into the groups when readers are bound in finalize().
"""
import logging

import numpy as np

from ..engine import bracket

logger = logging.getLogger('opendrift_b200')

# variables a StructuredReader serves without time interpolation (readers/basereader/structured.py:224-229)
STATIC_VARIABLES = ('sea_floor_depth_below_sea_level', 'land_binary_mask')

# drift:use_tabularised_stokes_drift (physics_methods.py:488-568): per fetch (m), the tabulated Stokes drift factor wf
# (Stokes drift = wf * wind) and significant wave height (m) at wind speeds 0, 1, ..., 29 m/s, and the order of the
# polynomial fitted to the Stokes drift factor (the height is fitted with a straight line)
STOKES_TABLES = {
    '5000': (3, (0.0173, 0.0160, 0.0152, 0.0145, 0.0139, 0.0135, 0.0132, 0.0129, 0.0126, 0.0124, 0.0122, 0.0121, 0.0119, 0.0118,
                 0.0117, 0.0116, 0.0114, 0.0113, 0.0112, 0.0112, 0.0111, 0.0110, 0.0109, 0.0109, 0.0108, 0.0107, 0.0106, 0.0106,
                 0.0106, 0.0105),
             (0.030, 0.077, 0.124, 0.170, 0.216, 0.263, 0.311, 0.360, 0.409, 0.459, 0.509, 0.560, 0.612, 0.664, 0.716, 0.771, 0.823,
              0.876, 0.932, 0.987, 1.041, 1.095, 1.152, 1.210, 1.265, 1.319, 1.375, 1.434, 1.494, 1.552)),
    '25000': (6, (0.0173, 0.0197, 0.0201, 0.0185, 0.0181, 0.0176, 0.0171, 0.0167, 0.0164, 0.0160, 0.0158, 0.0155, 0.0153, 0.0151,
                  0.0149, 0.0147, 0.0146, 0.0144, 0.0143, 0.0142, 0.0140, 0.0139, 0.0138, 0.0137, 0.0136, 0.0135, 0.0135, 0.0134,
                  0.0133, 0.0132),
              (0.030, 0.122, 0.251, 0.336, 0.442, 0.546, 0.650, 0.753, 0.856, 0.959, 1.063, 1.168, 1.273, 1.379, 1.486, 1.593, 1.702,
               1.811, 1.920, 2.030, 2.142, 2.254, 2.366, 2.478, 2.592, 2.707, 2.822, 2.936, 3.051, 3.166)),
    '50000': (6, (0.0173, 0.0197, 0.0210, 0.0216, 0.0201, 0.0194, 0.0190, 0.0186, 0.0183, 0.0179, 0.0176, 0.0173, 0.0171, 0.0168,
                  0.0166, 0.0164, 0.0162, 0.0160, 0.0159, 0.0157, 0.0156, 0.0155, 0.0153, 0.0152, 0.0151, 0.0150, 0.0149, 0.0148,
                  0.0147, 0.0146),
              (0.030, 0.122, 0.274, 0.474, 0.591, 0.724, 0.873, 1.021, 1.168, 1.314, 1.460, 1.606, 1.752, 1.898, 2.045, 2.192, 2.340,
               2.489, 2.639, 2.789, 2.940, 3.092, 3.244, 3.397, 3.551, 3.706, 3.862, 4.017, 4.173, 4.330)),
}


def stokes_coefficients(fetch):
    """(Stokes drift factor, significant wave height) polynomial coefficients for a fetch, highest power first: np.polyfit of
    the tables against the wind speed, in float64."""
    order, wf, hs = STOKES_TABLES[str(fetch)]
    return np.polyfit(range(len(wf)), wf, order), np.polyfit(range(len(hs)), hs, 1)


class Environment:
    def __init__(self, required_variables, config):
        self.required_variables = required_variables      # name -> spec dict
        self._config = config
        self.readers = {}
        self.priority_list = {}
        self.discarded_readers = {}
        self.__finalized__ = False
        self._engine = None
        self._stokes_coef = None          # (wf, Hs) coefficients while drift:use_tabularised_stokes_drift is on

    # -- registry (environment.py:267-330) -------------------------------------------------------
    def add_reader(self, readers, variables=None, first=False):
        if not isinstance(readers, (list, tuple)):
            readers = [readers]
        for r in readers:
            name = getattr(r, 'name', type(r).__name__)
            base, k = name, 1
            while name in self.readers:
                k += 1
                name = '%s_%d' % (base, k)
            r.name = name
            self.readers[name] = r
            for v in (variables or r.variables):
                if v not in r.variables:
                    continue
                lst = self.priority_list.setdefault(v, [])
                if first:
                    lst.insert(0, name)
                else:
                    lst.append(name)

    def finalize(self, engine):
        self._engine = engine
        ms = self._config._config.get('drift:max_speed')
        for r in self.readers.values():
            if hasattr(r, 'set_buffer_size') and ms is not None:
                r.set_buffer_size(max_speed=ms['value'])             # environment.py:402
            if hasattr(r, 'bind'):
                r.bind(engine, fallback={v: self.fallback(v) for v in r.variables})
        self._stokes_coef = None
        if self._config._config.get('drift:use_tabularised_stokes_drift', {}).get('value') is True:
            self._stokes_coef = stokes_coefficients(self._config.get_config('drift:tabularised_stokes_drift_fetch'))
        self.__finalized__ = True

    def subblock_readers(self):
        return [r for r in self.readers.values() if getattr(r, 'subblocks', False)]

    def ensure_windows(self, bbox, margin_deg):
        """Sub-block readers: their device blocks must cover the elements (bounding box + how far they can travel)."""
        return [r.ensure_window(bbox, margin_deg) for r in self.subblock_readers()]

    def touch_slabs(self, times):
        """Make every bound reader's slabs for the given times resident -- in a fixed order (readers as added, groups as bound,
        times as given).  In a distributed run this is where the slab collectives happen: every rank calls it at every step,
        whether it holds elements or not, so the ranks stay in lockstep; the step launches then find the slabs in place."""
        for r in self.readers.values():
            if not hasattr(r, '_groups'):
                continue
            seen = []
            for g, _ in r._groups.values():
                if any(g is x for x in seen):
                    continue
                seen.append(g)
                held = ()
                for t in times:
                    if r.covers_time(t):
                        _, q = g.sample(t, held)
                        held += q

    def constant(self, var):
        item = self._config._config.get('environment:constant:%s' % var)
        return None if item is None else item['value']

    def fallback(self, var):
        item = self._config._config.get('environment:fallback:%s' % var)
        return None if item is None else item['value']

    def discard_ended_readers(self, time):
        """Environment.discard_reader_if_not_relevant (environment.py:418-432), the rule that matters while a run is under
        way: a reader whose end_time lies before the requested time is discarded FOR GOOD ('ends before simulation is
        finished').  In a forward run that is indistinguishable from not covering the time any more; in a backward run that
        starts after the reader's end the reference never uses the reader again -- mirrored here."""
        for name, r in list(self.readers.items()):
            if getattr(r, 'start_time', None) is None or getattr(r, 'always_valid', False) or time is None:
                continue
            if r.end_time < time:
                self.discarded_readers[name] = 'ends before simuation is finished'
                del self.readers[name]
                for lst in self.priority_list.values():
                    if name in lst:
                        lst.remove(name)

    def reader_for(self, var, time):
        """First reader in priority order that provides `var` and covers `time` (or None)."""
        if self.constant(var) is not None:
            return None
        self.discard_ended_readers(time)
        for name in self.priority_list.get(var, []):
            r = self.readers[name]
            if r.covers_time(time):
                return r
        return None

    def readers_for(self, var, time):
        """All readers, in priority order, that provide `var` and cover `time` (the reference loops over them on the
        still-missing elements, environment.py:613-780)."""
        if self.constant(var) is not None:
            return []
        self.discard_ended_readers(time)
        return [self.readers[name] for name in self.priority_list.get(var, []) if self.readers[name].covers_time(time)]

    def readers_for_times(self, var, times):
        """Readers, in priority order, that provide `var` and cover at least ONE of `times` -- the stage times of a
        Runge-Kutta step (t, t + dt/2, t + dt): every get_environment call of the reference picks its readers for its own
        time, so a step that straddles the hand-over between two readers that follow each other in time uses both."""
        if self.constant(var) is not None:
            return []
        self.discard_ended_readers(times[0])       # the step's own time comes first; later stage times cannot add discards that matter
        return [self.readers[name] for name in self.priority_list.get(var, [])
                if any(self.readers[name].covers_time(t) for t in times)]

    # -- device face ---------------------------------------------------------------------------------
    def has_host_readers(self, variables=None):
        """True when a reader in the priority lists (of `variables`, or of all) computes its values on the host
        (readers/continuous.py): such a reader is sampled through device_sample(), never inside a fused launch."""
        for v, names in self.priority_list.items():
            if variables is not None and v not in variables:
                continue
            if any(getattr(self.readers.get(nm), 'host_callback', False) for nm in names):
                return True
        return False

    def has_ensembles(self, variables=None):
        """True when a gridded reader in the priority lists (of `variables`, or of all) serves ensemble blocks."""
        for v, names in self.priority_list.items():
            if variables is not None and v not in variables:
                continue
            for nm in names:
                r = self.readers.get(nm)
                if r is not None and hasattr(r, 'has_ensembles') and r.has_ensembles(v):
                    return True
        return False

    def device_environment(self, variables, time, d_lon, d_lat, d_z, pos_f32=False):
        """dict var -> float32 device tensor, with constants / fallbacks applied, + missing mask tensor."""
        eng = self._engine
        torch = eng.torch
        n = d_lon.numel()
        out = {}
        self.discard_ended_readers(time)
        for v in variables:
            if v in out:
                continue
            c = self.constant(v)
            if c is not None:
                out[v] = torch.full((n,), float(c), dtype=torch.float32, device=eng.device)
                continue
            res = None
            for name in self.priority_list.get(v, []):
                r = self.readers[name]
                if r.covers_time(time) and hasattr(r, 'device_sample'):      # analytical reader (no field group)
                    smp = r.device_sample(eng, time, d_lon, d_lat, pos_f32, d_z=d_z) if getattr(r, 'host_callback', False) \
                        else r.device_sample(eng, time, d_lon, d_lat, pos_f32)
                    if res is None:
                        res = dict(smp)
                    else:
                        for nm, t_ in smp.items():
                            if nm in res:
                                res[nm] = torch.where(torch.isfinite(res[nm]), res[nm], t_)
                    if bool(torch.isfinite(res[v]).all()):
                        break
                    continue
                if not r.covers_time(time) or not hasattr(r, 'group_of'):
                    continue
                g, comp = r.group_of(v)
                t_s, nearest = time, False
                if all(nm in STATIC_VARIABLES for nm, (gg, _) in r._groups.items() if gg is g):
                    # variables that do not depend on time are taken from the block before `time`, without the time lerp
                    # (structured.py:224-229); land_binary_mask from the nearest grid point (interpolation/structured.py:117-119)
                    br = bracket(g.times, time)
                    if br is not None:
                        t_s = g.times[br[0]]
                    nearest = v == 'land_binary_mask' and not getattr(r, 'always_valid', False)   # (a constant reader has one value everywhere)
                need = None if res is None or v not in res else ~torch.isfinite(res[v])     # the elements this reader is asked for
                outs = r.sample_groups(eng, v, t_s, d_lon, d_lat, d_z, need=need, pos_f32=pos_f32, raw=True, nearest=nearest)
                if res is None:
                    res = {nm: outs[cc] for nm, (gg, cc) in r._groups.items() if gg is g}
                else:                                   # next reader fills what is still missing
                    for nm, (gg, cc) in r._groups.items():
                        if gg is g and nm in res:
                            res[nm] = torch.where(torch.isfinite(res[nm]), res[nm], outs[cc])
                if bool(torch.isfinite(res[v]).all()):
                    break
            if res is None:
                res = {v: torch.full((n,), float('nan'), dtype=torch.float32, device=eng.device)}
            for nm, t in res.items():
                if nm in variables and nm not in out:
                    fb = self.fallback(nm)
                    if fb is not None:
                        t = torch.where(torch.isfinite(t), t, torch.full_like(t, float(fb)))
                    out[nm] = t
        if self._stokes_coef is not None and 'x_wind' in out:
            self._parameterise_stokes(out)
        missing = torch.zeros(n, dtype=torch.bool, device=eng.device)
        for v in variables:
            missing |= ~torch.isfinite(out[v])
        return out, missing

    def _parameterise_stokes(self, out):
        """drift:use_tabularised_stokes_drift (environment.py:844-863), after the fallbacks and before any uncertainty draw: both
        Stokes components become wind * wf when the maximum of each is exactly 0 over the call's elements (a reader whose values
        are all <= 0 with one exact 0 included), and Hs the fitted height when its maximum is 0.  A variable the call did not
        request is left out (the reference has no field to write it into and stops)."""
        eng, torch = self._engine, self._engine.torch
        sx, sy = 'sea_surface_wave_stokes_drift_x_velocity', 'sea_surface_wave_stokes_drift_y_velocity'
        hs = 'sea_surface_wave_significant_height'
        if 'y_wind' not in out:
            return
        stokes = sx in out and sy in out and eng.minmax(out[sx])[1] == 0 and eng.minmax(out[sy])[1] == 0
        height = hs in out and eng.minmax(out[hs])[1] == 0
        if not (stokes or height):
            return
        # fresh outputs: a sampled tensor may be shared with another variable or a reader
        us = torch.empty_like(out['x_wind']) if stokes else None
        vs = torch.empty_like(out['x_wind']) if stokes else None
        h = torch.empty_like(out['x_wind']) if height else None
        eng.stokes_parameterised(out['x_wind'], out['y_wind'], self._stokes_coef[0], self._stokes_coef[1], us, vs, h)
        if stokes:
            out[sx], out[sy] = us, vs
        if height:
            out[hs] = h

    # -- host face (the reference signature) ---------------------------------------------------------
    def get_environment(self, variables, time, lon, lat, z, profiles=None, profiles_depth=None, element_ID=None):
        assert self.__finalized__ is True, 'The environment has not been finalized.'
        eng = self._engine
        lon, lat = np.atleast_1d(lon), np.atleast_1d(lat)
        n = len(lon)
        pos_f32 = lon.dtype == np.float32 and lat.dtype == np.float32
        trunc = self._config.get_config('drift:truncate_ocean_model_below_m', None) \
            if 'drift:truncate_ocean_model_below_m' in self._config._config else None
        zz = np.asarray(z, dtype=np.float32) * np.ones(n, dtype=np.float32)
        if trunc is not None:
            zz = zz.copy()
            zz[zz < -trunc] = -trunc
        d_env, d_missing = self.device_environment(list(variables), time, eng.to_device(lon.astype(np.float64)),
                                                   eng.to_device(lat.astype(np.float64)), eng.to_device(zz), pos_f32)
        env = np.zeros(n, dtype=[(v, np.float32) for v in variables])
        for v in variables:
            env[v] = d_env[v].cpu().numpy()
        env_profiles = None
        if profiles:
            if profiles_depth is None:
                profiles_depth = np.abs(np.asarray(z)).max()       # (:552-553)
            if trunc is not None:
                profiles_depth = np.minimum(profiles_depth, trunc)
            env_profiles = self._host_profiles(list(profiles), profiles_depth, time, lon, lat, zz, env)
        return env.view(np.recarray), env_profiles, d_missing.cpu().numpy()

    def _host_profiles(self, profiles, profiles_depth, time, lon, lat, z, env):
        """The `profiles` part of get_environment (:627-640, 697-724, 793-822) for callers outside the step kernels (the vertical
        mixing launch reads the field column itself): per variable the layers of the first reader that provides it, down to the
        first level below profiles_depth; fallback values where that reader has nothing; `[value, value]` at `z = [0, -depth]` for
        a constant or a variable no reader provides.  Several readers filling one another's gaps layer by layer are refused."""
        from ..errors import NotCoveredError
        n = len(lon)
        out = {}
        for var in profiles:
            fb = self.fallback(var)
            readers = [self.readers[nm] for nm in self.priority_list.get(var, []) if self.readers[nm].covers_time(time)] \
                if self.constant(var) is None else []
            got = None
            for r in readers:
                try:
                    _, prof = r.get_variables_interpolated([var], profiles=[var], profiles_depth=profiles_depth, time=time, lon=lon, lat=lat, z=z)
                except NotCoveredError:
                    continue
                if got is not None:
                    raise NotImplementedError('profiles of %s from several readers that cover parts of the elements are not on the GPU path' % var)
                a = np.ma.masked_invalid(np.ma.atleast_2d(prof[var]))
                if np.ma.getmaskarray(a).any() and len(readers) > 1:
                    raise NotImplementedError('profiles of %s from several readers that cover parts of the elements are not on the GPU path' % var)
                got = (np.asarray(prof['z']), a)
            if got is None:
                zs = np.array([0, -profiles_depth])
                val = env[var] if (var in env.dtype.names and (self.constant(var) is not None or readers)) else (np.nan if fb is None else fb)
                a = np.ma.masked_invalid(np.ma.array([val * np.ones(n), val * np.ones(n)]))
                got = (zs, a)
            zs, a = got
            if 'z' in out and (len(out['z']) != len(zs) or not np.allclose(out['z'], zs)):
                raise NotImplementedError('profiles on different vertical levels (%s) are not on the GPU path' % var)
            out['z'] = zs
            data = np.array(np.ma.getdata(a), dtype=np.float64, copy=True)
            # (:699-718: the first reader's profile is stored and then written onto itself through float32, all layers but the last)
            data[:-1] = data[:-1].astype(np.float32)
            mask = np.ma.getmaskarray(a)
            if mask.any():
                data[mask] = np.nan if fb is None else fb
            out[var] = data
        return out
