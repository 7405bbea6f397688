"""Reader base classes with the reference's public surface for geographic regular-grid readers.

Mirrors, for `+proj=latlong` structured readers,
  opendrift/readers/basereader/variables.py  (ReaderDomain/Variables: coverage, nearest_time,
      get_variables_interpolated[_xy], valid-range check :630-668)
  opendrift/readers/basereader/structured.py (StructuredReader: before/after block cache, time interpolation)
  opendrift/readers/interpolation/structured.py + interpolators.py (ReaderBlock, linearNDFast + linear)
but the arithmetic runs in libodcuda.so: a reader is *bound* to an Engine, its blocks become device-resident
field groups (a ring of time slabs in HBM), and get_variables_interpolated() is a thin host wrapper around
od_interp (host arrays in, host arrays out, as the reference returns NumPy).  The fused step kernels use
the bound groups directly.

Reader implementers keep the reference contract (basereader/structured.py:125-147): provide
`get_variables(requested_variables, time, x, y, z)` returning {'x','y','z','time', var: ndarray[(z,)y,x]} and
the attributes proj4, xmin/xmax/ymin/ymax, variables, start_time/end_time/time_step (or times), name.
"""
import numpy as np

from ..errors import (NotCoveredError, OutsideSpatialCoverageError,  # noqa: F401
                      OutsideTemporalCoverageError, VariableNotCoveredError)

# valid (but extreme) ranges, opendrift/readers/basereader/consts.py:2-21
standard_names = {
    'x_wind': (-50, 50), 'y_wind': (-50, 50),
    'x_sea_water_velocity': (-15, 15), 'y_sea_water_velocity': (-15, 15),
    'land_binary_mask': (0, 1), 'sea_floor_depth_below_sea_level': (-20, 12000),
    'ocean_vertical_diffusivity': (0, 1)}

# x/y vector pairs that are always sampled together (consts.py:26-36)
vector_pairs_xy = [
    ('x_wind', 'y_wind'),
    ('sea_ice_x_velocity', 'sea_ice_y_velocity'),
    ('x_sea_water_velocity', 'y_sea_water_velocity'),
    ('sea_surface_wave_stokes_drift_x_velocity', 'sea_surface_wave_stokes_drift_y_velocity')]


def check_variable_array(name, a):
    """Variables.__check_variable_array__ (variables.py:630-668): masked -> NaN, out-of-range -> NaN."""
    if isinstance(a, np.ma.MaskedArray):
        a = a.astype(np.float32).filled(np.nan)
    a = np.array(a, dtype=np.float32, copy=True)
    if name in standard_names:
        lo, hi = standard_names[name]
        with np.errstate(invalid='ignore'):
            bad = np.isfinite(a) & ((a < lo) | (a > hi))
        if bad.any():
            a[bad] = np.nan
    return a


def fill_nan_towards_seafloor(a):
    """interpolators.py:204-212: copy layer i-1 into the NaNs of layer i."""
    for i in range(1, a.shape[0]):
        m = np.isnan(a[i])
        if m.any():
            a[i][m] = a[i - 1][m]
    return a


def check_arguments(self, variables, time, x, y, z):
    """variables.py:321-390 -- what reader classes written for the reference call first thing in get_variables: the variable
    list, the time (the reader's first when None), x / y as arrays, and the indices of positions outside the reader's domain;
    raises for unknown variables, times outside the coverage, and when every position is outside."""
    from ..errors import VariableNotCoveredError, OutsideTemporalCoverageError, OutsideSpatialCoverageError
    if time is None:
        time = self.start_time
    if isinstance(variables, str):
        variables = [variables]
    no_positions = x is None or y is None        # (a whole-grid request of this package: nothing to check in space)
    if not no_positions:
        x, y = np.atleast_1d(x), np.atleast_1d(y)
    if z is not None:
        z = np.asarray(z)
    for v in variables:
        if v not in self.variables:
            raise VariableNotCoveredError('Variable not available: ' + v + '\nAvailable parameters are: ' + str(self.variables))
    if self.start_time is not None and time < self.start_time and self.always_valid is False:
        raise OutsideTemporalCoverageError('Requested time (%s) is before first available time (%s) of %s' % (time, self.start_time, self.name))
    if self.end_time is not None and time > self.end_time and self.always_valid is False:
        raise OutsideTemporalCoverageError('Requested time (%s) is after last available time (%s) of %s' % (time, self.end_time, self.name))
    if no_positions:
        return variables, time, x, y, z, np.zeros(0, dtype=np.int64)
    bad = ~np.isfinite(x + y) | (y < self.ymin) | (y > self.ymax)
    if not self.global_coverage():
        bad |= (x < self.xmin) | (x > self.xmax)
    outside = np.where(bad)[0]
    if np.size(outside) == np.size(x):
        raise OutsideSpatialCoverageError('Argcheck: all %s particles (%.2f-%.2fE, %.2f-%.2fN) are outside domain of %s'
                                          % (np.size(x), x.min(), x.max(), y.min(), y.max(), self.name))
    return variables, time, x, y, z, outside


class StructuredReader:
    """Regular lon/lat(/z) grid reader whose interpolation runs on the GPU."""

    name = 'structured_reader'
    proj4 = '+proj=latlong'
    times = None
    always_valid = False
    # True: get_variables(variables, time, x, y, z) is asked for the positions to cover (the corners of the elements' bounding
    # box) and returns a SUB-BLOCK of the grid around them, with its own x / y axes (reader_netCDF_CF_generic.py:404-626);
    # needs numx / numy (the full grid: capacity of the device slots).  False: the reader hands out its whole grid.
    subblocks = False
    buffer = 0

    def __init__(self):
        p = str(getattr(self, 'proj4', '+proj=latlong'))
        # a projected plane (+proj=stere, +proj=merc, +proj=lcc): x / y axes and xmin .. ymax are metres in it; a rotated pole
        # (+proj=ob_tran +o_proj=longlat): they are rotated longitude / latitude in degrees
        self.proj = None
        from .projection import RotatedPole, is_geographic, make_projection
        if not is_geographic(p):
            self.proj = make_projection(p)             # raises for what the device code does not project
            if self.subblocks:
                raise NotImplementedError('sub-block readers on a projected plane are not on the GPU path')
            if isinstance(self.proj, RotatedPole):
                self._check_rotated_grid()
            # modulate_longitude (variables.py:259-280): the longitude convention follows the corner longitudes
            exlons, _ = self.proj(np.array([self.xmin, self.xmin, self.xmax, self.xmax], dtype=np.float64),
                                  np.array([self.ymin, self.ymax, self.ymax, self.ymin], dtype=np.float64), inverse=True)
            self._lon_0to360 = not (np.min(exlons) < 0)
        if getattr(self, 'times', None) is None and getattr(self, 'start_time', None) is not None \
                and getattr(self, 'time_step', None) is not None and self.end_time != self.start_time:
            n = int(round((self.end_time - self.start_time).total_seconds() / self.time_step.total_seconds())) + 1
            self.times = [self.start_time + i * self.time_step for i in range(n)]
        elif getattr(self, 'times', None) is None:
            self.times = [self.start_time]
        self.zmin, self.zmax = -np.inf, np.inf
        self._engine = None
        self._groups = {}          # variable -> (FieldGroup, component)
        self._block_geom = None
        self.number_of_fails = 0
        self._request = None       # sub-block readers: (x, y) corner positions of the current block request
        self._window = None        # ... and the extent (xmin, xmax, ymin, ymax) of the block that came back
        self._block_caches = []
        self.windows_set = 0

    def _check_rotated_grid(self):
        """A rotated-pole grid that the reference would treat as global east-west (variables.py:289-301: it tests the rotated
        axis as if it were longitude), or whose y-axis line of rotate_vectors (0.1 degrees north in the rotated plane) could cross
        the rotated pole, is refused."""
        dx = getattr(self, 'delta_x', None) or 0
        if (self.xmin - 2 * dx <= 0 and self.xmax + 2 * dx >= 360) or (self.xmin - 2 * dx <= -180 and self.xmax + 2 * dx >= 180):
            raise NotImplementedError('a rotated-pole grid spanning 360 degrees of rotated longitude is not on the GPU path')
        if self.ymax + 0.1 >= 90 or self.ymin - 0.1 <= -90:
            raise NotImplementedError('a rotated-pole grid within 0.1 degrees of the rotated pole is not on the GPU path')

    # -- coverage (variables.py:229-257, 391-400) ------------------------------------------------
    def covers_time(self, time):
        if self.start_time is None:
            return True
        return self.start_time <= time <= self.end_time

    def modulate_longitude(self, lons):
        lons = np.asarray(lons)
        if self.proj is not None:
            return np.mod(lons, 360) if self._lon_0to360 else np.mod(lons + 180, 360) - 180
        return np.mod(lons + 180, 360) - 180 if self.xmin < 0 else np.mod(lons, 360)

    def lonlat2xy(self, lon, lat):
        """variables.py:129-143"""
        return (lon, lat) if self.proj is None else self.proj(lon, lat, inverse=False)

    def xy2lonlat(self, x, y):
        """variables.py:114-127"""
        return (x, y) if self.proj is None else self.proj(x, y, inverse=True)

    def global_coverage(self):
        """True if the reader covers the globe east-west (variables.py:289-301)."""
        if self.proj is not None:
            return False
        dx = getattr(self, 'delta_x', None) or 0
        return bool((self.xmin - 2 * dx <= 0 and self.xmax + 2 * dx >= 360) or
                    (self.xmin - 2 * dx <= -180 and self.xmax + 2 * dx >= 180))

    def lon_range(self):
        if not self.global_coverage():
            raise ValueError('Only valid for readers with global coverage')
        return '-180to180' if self.xmin < 0 else '0to360'

    def covers_positions(self, lon, lat, z=0):
        x = self.modulate_longitude(np.atleast_1d(lon))
        y = np.atleast_1d(lat)
        if self.proj is not None:
            x, y = self.lonlat2xy(x, y)
        if self.global_coverage():             # north-south only (variables.py:239-242)
            ind = np.where((y >= self.ymin) & (y <= self.ymax))[0]
        else:
            # a rotated pole is geographic to pyproj: its rotated x is tested after modulate_longitude, whose convention comes
            # from the TRUE corner longitudes (variables.py:244-247, 259-280) -- an element can fall outside a grid it lies on
            xx = self.modulate_longitude(x) if self._rotated() else x
            ind = np.where((xx >= self.xmin) & (xx <= self.xmax) & (y >= self.ymin) & (y <= self.ymax))[0]
        return ind, x[ind], y[ind]

    def check_arguments(self, variables, time, x, y, z):
        return check_arguments(self, variables, time, x, y, z)

    def nearest_time(self, time):
        from ..engine import bracket
        br = bracket(self.times, time)
        if br is None:
            return None, None, None, None, None, None
        ib, ia, w = br
        tb = self.times[ib]
        ta = None if ia is None else self.times[ia]
        near = tb if (ta is None or (time - tb) < (ta - time)) else ta
        return near, tb, ta, self.times.index(near), ib, ia

    # -- block size (variables.py:154-165, 588-620) ---------------------------------------------------
    def pixel_size(self):
        dx = getattr(self, 'delta_x', None)
        if dx is None:
            return None
        return dx if self.proj is not None and not self._rotated() else dx * 111000   # degrees -> metres (also rotated degrees)

    def _rotated(self):
        from .projection import RotatedPole
        return isinstance(self.proj, RotatedPole)

    def set_buffer_size(self, max_speed, time_coverage=None):
        """Cells added around the requested positions so that the block still covers the elements at the end of the
        reader's time step: ceil(max_speed * time_step / pixel) + 2."""
        self.buffer = 0
        px = self.pixel_size()
        if px is not None:
            ts = getattr(self, 'time_step', None)
            secs = ts.total_seconds() if ts is not None else (3600 if time_coverage is None else time_coverage.total_seconds())
            self.buffer = int(np.ceil(max_speed * abs(secs) / px)) + 2

    # -- device binding --------------------------------------------------------------------------
    def _fetch_block(self, names, ti):
        """One reader block for time index ti via the reader's own get_variables(): the whole grid, or -- sub-block readers --
        the block around the current request (the corners of the elements' bounding box)."""
        t = self.times[ti]
        if self.subblocks and self._request is not None:
            x, y = self._request
            return self.get_variables(list(names), time=t, x=x, y=y, z=None)
        return self.get_variables(list(names), time=t, x=None, y=None, z=None)

    def ensure_window(self, bbox, margin_deg):
        """Sub-block readers: make the device blocks cover the elements' bounding box (lon min, lon max, lat min, lat max) grown
        by margin_deg (how far an element can travel before the next check).  When the current window does not, a new block is
        requested for the box -- the reader adds its own buffer (set_buffer_size) -- and its axes become the groups' index
        geometry; the ring refills on demand, the next slab ahead of time on the copy stream.  Returns True when re-windowed."""
        if not self.subblocks or self._engine is None or not np.all(np.isfinite(bbox)):
            return False
        x0, x1 = self.modulate_longitude(np.array([bbox[0], bbox[1]], dtype=np.float64))
        if x1 < x0:                                            # the box straddles the reader's longitude seam: whole rows
            x0, x1 = self.xmin, self.xmax
        y0, y1 = bbox[2], bbox[3]
        w = self._window
        inside = w is not None and (max(x0 - margin_deg, self.xmin) >= w[0] and min(x1 + margin_deg, self.xmax) <= w[1] and
                                    max(y0 - margin_deg, self.ymin) >= w[2] and min(y1 + margin_deg, self.ymax) <= w[3])
        if inside:
            return False
        self._request = (np.array([np.clip(x0, self.xmin, self.xmax), np.clip(x1, self.xmin, self.xmax)]),
                         np.array([np.clip(y0, self.ymin, self.ymax), np.clip(y1, self.ymin, self.ymax)]))
        for cache in self._block_caches:
            cache.clear()
        probe = self._fetch_block(self.variables[:1], 0)
        bx, by = np.asarray(probe['x'], dtype=np.float32), np.asarray(probe['y'], dtype=np.float32)
        self._window = (float(bx.min()), float(bx.max()), float(by.min()), float(by.max()))
        for g in {id(g): g for g, _ in self._groups.values()}.values():
            g.set_window(bx, by)
        self.windows_set += 1
        return True

    def bind(self, engine, fallback=None, n_slots=3):
        """Create the device field groups of this reader on `engine` (idempotent)."""
        if self._engine is engine:
            if fallback is not None:          # already bound (an earlier query, another model): follow this run's fallbacks
                for g in {id(g): g for g, _ in self._groups.values()}.values():
                    g.set_fallback([fallback.get(nme) for nme in g.names])
            return
        self._engine = engine
        self._groups = {}
        fallback = fallback or {}
        if self.subblocks:
            # the slots are sized for the whole grid (numx x numy: any window fits); the first probe only asks for one corner --
            # vertical levels and dimensionality of the variables -- the first real window comes with ensure_window()
            self._request = (np.array([self.xmin, self.xmin]), np.array([self.ymin, self.ymin]))
            self._window = None
        probe = self._fetch_block(self.variables, 0)
        x = np.asarray(probe['x'], dtype=np.float32)      # __check_env_coordinates__ (variables.py:622-628)
        y = np.asarray(probe['y'], dtype=np.float32)
        if self.subblocks:
            # the reader's full axes (only their length and end points matter here: capacity, longitude convention, coverage)
            fx, fy = getattr(self, 'lon', None), getattr(self, 'lat', None)
            x = np.asarray(fx, dtype=np.float32) if fx is not None and np.ndim(fx) == 1 and len(fx) == self.numx else \
                (self.xmin + self.delta_x * np.arange(self.numx)).astype(np.float32)
            y = np.asarray(fy, dtype=np.float32) if fy is not None and np.ndim(fy) == 1 and len(fy) == self.numy else \
                (self.ymin + self.delta_y * np.arange(self.numy)).astype(np.float32)
        done = set()
        plan = []
        for a, b in vector_pairs_xy:
            if a in self.variables and b in self.variables:
                plan.append((a, b))
                done |= {a, b}
        plan += [(v,) for v in self.variables if v not in done]
        self._ens = {}
        for names in plan:
            # Ensemble blocks: get_variables() returns a LIST of arrays for a variable, one per ensemble member, and element i of
            # a call is served by member i % n_members (ReaderBlock.interpolate, interpolation/structured.py:120-134).  Every member
            # becomes a field group of its own; Reader.sample_groups() picks the member per element.  (Not filled towards the sea
            # floor: 'Ensemble data currently not extrapolated towards seafloor', interpolation/structured.py:62-63.)
            ens = isinstance(probe[names[0]], (list, tuple))
            n_ens = len(probe[names[0]]) if ens else 1
            first = probe[names[0]][0] if ens else probe[names[0]]
            three_d = np.ndim(first) == 3
            z = np.asarray(probe['z'], dtype=np.float64) if three_d else None
            raw = {}                         # the reader's block of the time index in use, shared by the members
            groups = []
            for m in range(n_ens):
                cache = {}
                self._block_caches.append(cache)
                if m == 0:
                    self._block_caches.append(raw)

                def supplier(ti, c, names=names, cache=cache, raw=raw, m=m, ens=ens):
                    if ti not in cache:
                        cache.clear()
                        if ti not in raw:
                            raw.clear()
                            raw[ti] = self._fetch_block(names, ti)
                        blk = raw[ti]
                        arrs = []
                        for nme in names:
                            a = blk[nme][m] if ens else blk[nme]
                            if hasattr(a, 'is_cuda'):           # already a device tensor: trusted, no host pass
                                arrs.append(a)
                                continue
                            a = check_variable_array(nme, a)
                            if a.ndim == 3 and not ens:
                                fill_nan_towards_seafloor(a)
                            arrs.append(a)
                        cache[ti] = arrs
                    return cache[ti][c]
                fb = [fallback.get(nme) for nme in names]
                pk = {}
                if self.proj is not None:       # the block's axes are metres in the reader's plane; vector pairs get rotated
                    pk = dict(proj=self.proj.desc(), lon_0to360=self._lon_0to360, rotate=len(names) == 2)
                groups.append(engine.add_group(x, y, z, len(names), self.times, supplier, fb, n_slots=n_slots, names=names, **pk))
            for c, nme in enumerate(names):
                self._groups[nme] = (groups[0], c)
                if ens:
                    self._ens[nme] = groups

    def unbind(self):
        """Release the device slabs of this reader."""
        eng = self._engine
        if eng is not None:
            allg = [g for g, _ in self._groups.values()] + [g for gs in getattr(self, '_ens', {}).values() for g in gs]
            for g in {id(g): g for g in allg}.values():
                try:
                    eng.free_group(g)
                except Exception:
                    pass
        self._engine, self._groups, self._ens = None, {}, {}

    def __del__(self):
        try:
            self.unbind()
        except Exception:
            pass

    def group_of(self, variable):
        return self._groups[variable]

    def has_ensembles(self, variable=None):
        e = getattr(self, '_ens', {})
        return bool(e) if variable is None else variable in e

    def sample_groups(self, eng, v, t, d_lon, d_lat, d_z, need=None, **kw):
        """eng.interp for the field group of variable v.  Ensemble readers: every member group is sampled and element i of the
        positions THIS CALL SERVES -- those flagged in `need` (device bool tensor; None = all) that the reader covers -- takes
        member i % n_members (ReaderBlock.interpolate is handed exactly those positions, interpolation/structured.py:120-134;
        variables.py:709-858 passes the covered ones, environment.py:613-780 the still missing ones)."""
        g, _ = self._groups[v]
        members = getattr(self, '_ens', {}).get(v)
        if not members:
            return eng.interp(g, t, d_lon, d_lat, d_z, **kw)
        torch = eng.torch
        n = d_lon.numel()
        ind, _, _ = self.covers_positions(d_lon.cpu().numpy(), d_lat.cpu().numpy())
        served = torch.zeros(n, dtype=torch.bool, device=d_lon.device)
        served[eng.to_device(np.asarray(ind, dtype=np.int64))] = True
        if need is not None:
            served &= need
        member = (torch.cumsum(served.to(torch.int64), 0) - 1) % len(members)
        outs = None
        for m, gm in enumerate(members):
            om = eng.interp(gm, t, d_lon, d_lat, d_z, **kw)
            if outs is None:
                outs = [torch.full_like(o, float('nan')) for o in om]
            sel = served & (member == m)
            outs = [torch.where(sel, o, acc) for o, acc in zip(om, outs)]
        return outs

    # -- the reference's public entry point (variables.py:860-920) -----------------------------------
    def get_variables_interpolated(self, variables, profiles=None, profiles_depth=None, time=None,
                                   lon=None, lat=None, z=None, rotate_to_proj=None):
        if isinstance(variables, str):
            variables = [variables]
        assert set(variables).issubset(self.variables), f'{variables} is not subset of {self.variables}'
        if profiles is not None and isinstance(profiles, str):
            profiles = [profiles]
        if not self.covers_time(time):
            raise OutsideTemporalCoverageError('%s is outside time coverage (%s - %s) of %s'
                                               % (time, self.start_time, self.end_time, self.name))
        if self._engine is None:
            from ..engine import default_engine
            self.bind(default_engine())
        eng = self._engine
        lon_in, lat_in = np.atleast_1d(lon), np.atleast_1d(lat)
        n = len(lon_in)
        pos_f32 = lon_in.dtype == np.float32 and lat_in.dtype == np.float32
        ind, xc, yc = self.covers_positions(lon_in, lat_in)
        if len(ind) == 0:
            raise OutsideSpatialCoverageError('All %s particles are outside domain of %s' % (n, self.name))
        if self.subblocks:
            # the block around the positions this call is about (structured.py:275-318 asks its reader for exactly that); a model
            # run has done this for the elements' bounding box already (_cover_elements_with_blocks) and the window then holds
            self.ensure_window((float(np.min(xc)), float(np.max(xc)), float(np.min(yc)), float(np.max(yc))), 0.0)
        # (the depths keep their dtype: the reference clips and interpolates a float64 z in float64, interpolators.py:174-197)
        if z is None:
            zz = np.zeros(n, dtype=np.float32)
        else:
            zz = np.atleast_1d(np.asarray(z))
            zz = (zz.astype(np.float64) if zz.dtype == np.float64 else zz.astype(np.float32)) * np.ones(n, dtype=zz.dtype if zz.dtype == np.float64 else np.float32)
        d_lon = eng.to_device(lon_in.astype(np.float64))
        d_lat = eng.to_device(lat_in.astype(np.float64))
        d_z = eng.to_device(zz)
        env = {}
        for v in variables:
            if v in env:
                continue
            g, c = self._groups[v]
            # no fallback here: uncovered / missing samples are NaN-masked like the reference's reader output
            # (a projected reader's vector pairs are rotated to east / north when the caller names the target CRS, as
            # Environment does with rotate_to_proj = '+proj=latlong'; without it the components stay along the grid's axes)
            # the reference returns float64 for 3-D blocks -- the unrounded vertical and time lerp (interpolation/structured.py:139-140,
            # basereader/structured.py:353-364) -- and float32 for 2-D blocks; land_binary_mask comes from the nearest grid point and,
            # like the sea floor depth, from the block before `time` without a time lerp (structured.py:224-229)
            three_d = g.desc.nz > 1
            names = [nme for nme, (gg, _) in self._groups.items() if gg is g]
            t_s, nearest = time, False
            if all(nme in ('sea_floor_depth_below_sea_level', 'land_binary_mask') for nme in names):
                from ..engine import bracket
                br = bracket(g.times, time)
                if br is not None:
                    t_s = g.times[br[0]]
                nearest = v == 'land_binary_mask' and not getattr(self, 'always_valid', False)   # (a constant reader has one value everywhere)
            # (a rotated vector pair is float64 also for 2-D blocks: rotate_vectors multiplies by float64 sines and cosines)
            rotated = self.proj is not None and rotate_to_proj is not None and len(names) == 2
            outs = self.sample_groups(eng, v, t_s, d_lon, d_lat, d_z, pos_f32=pos_f32, raw=True, rotate=rotate_to_proj is not None,
                                      out_f64=three_d or rotated, nearest=nearest)
            for nme, (gg, cc) in self._groups.items():
                if gg is g and nme in variables:
                    a = outs[cc].cpu().numpy()
                    if len(ind) != n:          # some positions are not covered: the reference pads into a float64 array (variables.py:841-846)
                        a = a.astype(np.float64)
                    env[nme] = np.ma.masked_invalid(a)
        env_profiles = None
        if profiles:
            # Vertical profiles (interpolation/structured.py:137-138, basereader/structured.py:365-384): for every requested variable
            # the horizontally interpolated value of EVERY layer of the block, (nz, N), float64, lerped in time like the values --
            # one sampling launch per layer at the layer's own depth (the vertical lerp then has weight 1 on that layer).  The run
            # loop does not use this call (the mixing kernel walks the columns itself); it serves user code.
            env_profiles = {}
            for v in profiles:
                g, c = self._groups[v]
                if g.desc.nz <= 1:
                    raise NotImplementedError('profiles of a 2-D variable (%s)' % v)
                zl = np.asarray(g.z, dtype=np.float64)          # the levels as the reader gave them
                env_profiles.setdefault('z', zl)
                rows = []
                for zk in zl:
                    d_zk = eng.to_device(np.full(n, zk, dtype=np.float64))
                    outs = eng.interp(g, time, d_lon, d_lat, d_zk, pos_f32=pos_f32, raw=True, rotate=rotate_to_proj is not None, out_f64=True)
                    rows.append(outs[c].cpu().numpy())
                env_profiles[v] = np.ma.masked_invalid(np.stack(rows))
        return env, env_profiles

    def __repr__(self):
        return 'Reader: %s  [%s..%s] x [%s..%s], %s - %s, variables %s' % (
            self.name, self.xmin, self.xmax, self.ymin, self.ymax, self.start_time, self.end_time, self.variables)
