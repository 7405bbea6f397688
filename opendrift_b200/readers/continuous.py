"""ContinuousReader: the reference's extension point for analytical readers (opendrift/readers/basereader/continuous.py) -- a subclass
provides `get_variables(variables, time, x, y, z)` returning exact values AT the positions it is given, no grid, no time lerp.

User code of that kind is host code (NumPy): the positions of the elements it is asked about are copied to the host, the subclass's
`get_variables` runs as it would under the reference -- same arguments: the reader's own longitude convention, float32 positions on
a run's first step, the elements' depths --, and the values go back to the device as float32, NaN where the reader does not cover a
position.  Every sample is a round trip over PCIe, so a model with such a reader takes the helper / staged recipes (one round trip per
Runge-Kutta stage), not the fused step kernels; the analytical reader of BASELINE configs[0] (reader_double_gyre) is evaluated on the
device instead (csrc/od_analytic.cuh)."""
import numpy as np

from ..errors import OutsideSpatialCoverageError


class ContinuousReader:
    always_valid = False
    host_callback = True        # Environment / the model recipes: sampled through device_sample(), never inside a fused launch
    name = 'continuous_reader'
    proj4 = '+proj=latlong'
    xmin, xmax, ymin, ymax = -180, 180, -90, 90
    start_time = end_time = time_step = None

    def __init__(self):
        p = str(getattr(self, 'proj4', '+proj=latlong'))
        from .projection import is_geographic
        if not is_geographic(p):                   # (a rotated pole, +o_proj=longlat, is not geographic)
            raise NotImplementedError('ContinuousReader subclasses on a projected plane are not on the GPU path (got %r); the '
                                      'projected analytical reader that is: readers/reader_double_gyre.py' % p)
        self.zmin, self.zmax = -np.inf, np.inf
        self._engine = None

    def get_variables(self, variables, time=None, x=None, y=None, z=None):
        raise NotImplementedError('a ContinuousReader subclass provides get_variables(variables, time, x, y, z)')

    # -- coverage (variables.py:229-280, 391-400) --------------------------------------------------------------
    def covers_time(self, time):
        if self.start_time is None:
            return True
        return self.start_time <= time <= self.end_time

    def modulate_longitude(self, lons):
        lons = np.asarray(lons)
        return np.mod(lons + 180, 360) - 180 if self.xmin < 0 else np.mod(lons, 360)

    def lonlat2xy(self, lon, lat):
        return lon, lat

    def xy2lonlat(self, x, y):
        return x, y

    def global_coverage(self):
        return bool((self.xmin <= 0 and self.xmax >= 360) or (self.xmin <= -180 and self.xmax >= 180))

    def covers_positions(self, lon, lat, z=0):
        x, y = self.modulate_longitude(np.atleast_1d(lon)), np.atleast_1d(lat)
        ind = np.where((x >= self.xmin) & (x <= self.xmax) & (y >= self.ymin) & (y <= self.ymax))[0]
        return ind, x[ind], y[ind]

    def check_arguments(self, variables, time, x, y, z):
        from .basereader import check_arguments
        return check_arguments(self, variables, time, x, y, z)

    # -- device binding ----------------------------------------------------------------------------------------
    def bind(self, engine, fallback=None):
        self._engine = engine

    def unbind(self):
        self._engine = None

    def _sample_host(self, variables, time, lon, lat, z):
        """{variable: float32 array, NaN where uncovered} for host arrays (variables.py:709-858 without the rotation: the
        reader's plane is the geographic one)."""
        n = len(lon)
        ind, x, y = self.covers_positions(lon, lat)
        out = {v: np.full(n, np.nan, dtype=np.float32) for v in variables}
        if len(ind) == 0:
            return out
        if z is None:
            zc = None
        else:
            z = np.asarray(z)
            zc = z[ind] if z.ndim and len(z) == n else z
        env = self.get_variables(list(variables), time, x, y, zc)
        for v in variables:
            out[v][ind] = np.ma.filled(np.ma.masked_invalid(np.asarray(env[v], dtype=np.float64) * np.ones(len(ind))), np.nan)
        return out

    def device_sample(self, engine, time, d_lon, d_lat, pos_f32=False, d_z=None):
        """{variable: float32 device tensor}, NaN where the reader does not cover the position (no fallback)."""
        lon, lat = d_lon.cpu().numpy(), d_lat.cpu().numpy()
        if pos_f32:                 # a run's first step: the reference hands the float32 positions of the seeding on
            lon, lat = lon.astype(np.float32), lat.astype(np.float32)
        z = None if d_z is None else d_z.cpu().numpy()
        out = self._sample_host(self.variables, time, lon, lat, z)
        return {v: engine.to_device(a) for v, a in out.items()}

    # -- the reference's public entry point (basereader/variables.py:860-920) ---------------------------------
    def get_variables_interpolated(self, variables, profiles=None, profiles_depth=None, time=None,
                                   lon=None, lat=None, z=None, rotate_to_proj=None):
        if isinstance(variables, str):
            variables = [variables]
        assert set(variables).issubset(self.variables), f'{variables} is not subset of {self.variables}'
        lon, lat = np.atleast_1d(lon), np.atleast_1d(lat)
        out = self._sample_host(variables, time, lon, lat, None if z is None else np.atleast_1d(z))
        env = {v: np.ma.masked_invalid(out[v]) for v in variables}
        if all(np.ma.getmaskarray(a).all() for a in env.values()):
            raise OutsideSpatialCoverageError('All %s particles are outside domain of %s' % (len(lon), self.name))
        env_profiles = None
        if profiles is not None:                 # continuous.py:40-46: the value itself at both ends of the profile
            env_profiles = {'z': [0, -profiles_depth]}
            for var in profiles:
                env_profiles[var] = np.ma.array([env[var], env[var]])
        return env, env_profiles

    def __repr__(self):
        return 'Reader: %s (continuous; values computed on the host)' % self.name
