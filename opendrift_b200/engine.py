"""Thin Python owner of one od_ctx (one per GPU / process): field groups, slab residency and
the kernel calls.  PyTorch is used only to allocate device buffers and to provide the CUDA
stream; every computation happens in libodcuda.so.

Host logic restated from the reference:
  * which reader time slabs bracket a requested time, and the interpolation weight
    (Variables.nearest_time, opendrift/readers/basereader/variables.py:402-443;
    StructuredReader._get_variables_interpolated_, readers/basereader/structured.py:218-229, 353-356);
  * the before/after block cache with swap-on-advance (structured.py:243-318) becomes a ring of
    device-resident slabs per field group.
"""
import ctypes as C
import gc
import weakref
from bisect import bisect_left

import numpy as np

from . import _lib
from ._lib import (GroupDesc, TimeSample, AdvectArgs, StepArgs, MixArgs, StokesArgs, LeewayArgs, OD_T_LERP, OD_T_FIRST,
                   OD_T_MISSING, SCHEMES)


def _seconds(t, t0):
    return (t - t0).total_seconds() if hasattr(t - t0, 'total_seconds') else float(t - t0)


def bracket(times, t):
    """(index_before, index_after_or_None, weight_after) of time t in the sorted list `times`.

    Follows Variables.nearest_time for readers with a `times` list (variables.py:414-430) and the
    `time == time_before -> no after block` rule (structured.py:224-229); returns None when t is
    outside the reader's time coverage (covers_time, variables.py:391-400)."""
    if len(times) == 1:
        return 0, None, 0.0
    if t < times[0] or t > times[-1]:
        return None
    ib = max(0, bisect_left(times, t) - 1)
    if times[ib + 1] == t:
        ib += 1
    tb = times[ib]
    if t == tb:
        return ib, None, 0.0
    ia = min(ib + 1, len(times) - 1)
    ta = times[ia]
    w = _seconds(t, tb) / _seconds(ta, tb)
    return ib, ia, w


def draw_uncertainty(n, scheme, cur_std=0.0, cur_uniform=0.0, wind_std=0.0, with_wind=False, stage0=None):
    """The uncertainty draws of one time step from NumPy's legacy global generator, in the reference's order
    (environment.py:869-891, called once for the step's environment and once per Runge-Kutta stage):
    returns (noise_cur [4][2][2][n] float64 or None, kinds bitmask, noise_wind [2][n] or None)."""
    kinds = (1 if cur_std > 0 else 0) | (2 if cur_uniform > 0 else 0)
    stages = {'euler': 1, 'runge-kutta': 2, 'runge-kutta4': 4}[scheme]
    cur = np.zeros((4, 2, 2, n)) if kinds else None
    wind = None
    for st in range(stages):
        if st == 0 and stage0 is not None:
            # the step's own environment was drawn when the reference draws it: before this step's deactivations and
            # removals (basemodel/__init__.py:2238-2262), for the elements that were active then
            if cur_std > 0:
                cur[0, 0, 0], cur[0, 0, 1] = stage0['cur_n']
            if cur_uniform > 0:
                cur[0, 1, 0], cur[0, 1, 1] = stage0['cur_u']
            if with_wind and wind_std > 0:
                wind = np.stack(stage0['wind'])
            continue
        if cur_std > 0:
            cur[st, 0, 0] = np.random.normal(0, cur_std, n)
            cur[st, 0, 1] = np.random.normal(0, cur_std, n)
        if cur_uniform > 0:
            cur[st, 1, 0] = np.random.uniform(-cur_uniform, cur_uniform, n)
            cur[st, 1, 1] = np.random.uniform(-cur_uniform, cur_uniform, n)
        if st == 0 and with_wind and wind_std > 0:
            wind = np.stack([np.random.normal(0, wind_std, n), np.random.normal(0, wind_std, n)])
    return cur, kinds, wind


def _ptr(t):
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def grid_geometry(lon, lat):
    """What the sampler needs to know about a regular float32 lon/lat grid, following the reference:
    * Linear2DInterpolator (interpolators.py:110-111): xi = (x - xg[0]) / (xg[-1] - xg[0]) * (nx - 1), float32 end points and
      float32 difference;
    * longitude convention of the reader (variables.py:259-280): [-180, 180) when the grid starts west of 0, else [0, 360);
    * east-west global coverage (variables.py:289-301).  A global grid that is exactly periodic (nx * dx == 360) is sampled
      as the block 'all columns + column 0 again at lon[-1] + dx' (include/odcuda.h: wrap_x), which covers the seam cell."""
    lon = np.asarray(lon, dtype=np.float32)
    lat = np.asarray(lat, dtype=np.float32)
    xmin, xmax = float(lon.min()), float(lon.max())
    dx = float(lon[1] - lon[0])
    glob = (xmin - 2 * dx <= 0 and xmax + 2 * dx >= 360) or (xmin - 2 * dx <= -180 and xmax + 2 * dx >= 180)
    periodic = bool(glob) and abs(len(lon) * dx - 360.0) < 1e-3 * dx
    x_last = np.float32(lon[-1] + np.float32(dx)) if periodic else lon[-1]
    return {'lon_mode': _lib.OD_LON_PM180 if xmin < 0 else _lib.OD_LON_0_360, 'wrap_x': 1 if periodic else 0, 'global_x': 1 if glob else 0,
            'global_coverage': bool(glob),
            'x0': float(lon[0]), 'xspan': float(np.float32(x_last - lon[0])),
            'y0': float(lat[0]), 'yspan': float(np.float32(lat[-1] - lat[0])),
            'xmin': xmin, 'xmax': xmax, 'ymin': float(lat.min()), 'ymax': float(lat.max())}


class FieldGroup:
    """One od group: geometry + a ring of device slots filled on demand from a slab supplier."""

    def __init__(self, engine, gid, lon, lat, z, ncomp, times, supplier, fallback, n_slots=3,
                 names=None, proj=None, lon_0to360=False, rotate=False):
        self.engine, self.gid, self.ncomp = engine, gid, ncomp
        self.lon = np.asarray(lon, dtype=np.float32)
        self.lat = np.asarray(lat, dtype=np.float32)
        self.z = None if z is None else np.asarray(z, dtype=np.float64)
        self.times = list(times)
        self.supplier = supplier          # supplier(time_index, comp) -> float32 [nz,]ny,nx (NumPy or CUDA tensor)
        self.names = names
        self.n_slots = n_slots
        self.freed = False
        self.fill_nan = 10                # passes of the linearNDFast NaN fill applied to every uploaded slab (0 = off)
        self.resident = [None] * n_slots  # time index held by each ring slot
        self.use = [0] * n_slots
        self.ready = [None] * n_slots     # event of a slab that was put into its slot on the copy stream (prefetch), until first use
        self.prefetch_on = True
        self._tick = 0
        d = GroupDesc()
        d.ncomp, d.nx, d.ny = ncomp, len(self.lon), len(self.lat)
        d.nz = 1 if self.z is None else len(self.z)
        d.n_slots = n_slots
        geo = grid_geometry(self.lon, self.lat)
        if proj is not None:
            # the axes are metres in a projected plane: no longitude conventions of the axes, no periodicity; the longitude of
            # the positions is modulated as the reader's corner longitudes say, then projected (od_group_desc.proj)
            geo.update(lon_mode=_lib.OD_LON_0_360 if lon_0to360 else _lib.OD_LON_PM180, wrap_x=0, global_x=0, global_coverage=False)
            d.proj = proj
            d.rotate_vectors = 1 if (rotate and ncomp == 2) else 0
        d.lon_mode, d.wrap_x, d.global_x = geo['lon_mode'], geo['wrap_x'], geo['global_x']
        d.x0, d.xspan, d.y0, d.yspan = geo['x0'], geo['xspan'], geo['y0'], geo['yspan']
        d.xmin, d.xmax, d.ymin, d.ymax = geo['xmin'], geo['xmax'], geo['ymin'], geo['ymax']
        self.global_coverage, self.periodic = geo['global_coverage'], bool(geo['wrap_x'])
        fb = list(fallback) + [float('nan')] * (2 - len(fallback))
        d.fallback[0] = float('nan') if fb[0] is None else fb[0]
        d.fallback[1] = float('nan') if fb[1] is None else fb[1]
        self.desc = d
        zl = None
        if self.z is not None:
            zl = (C.c_double * len(self.z))(*self.z)
        engine._check(engine.lib.od_group_define(engine.ctx, gid, C.byref(d), zl))

    def set_window(self, lon, lat):
        """The blocks of this group now cover the window of the reader's grid with the axes lon, lat (float32, as the reader's
        block hands them out): block-relative index geometry as ReaderBlock's interpolator would form it, every ring slot
        invalidated.  The reader's own coverage (xmin .. ymax of the descriptor) is unchanged: an element inside the reader's domain
        but outside the block gets the block's edge value, as the reference's NaN loop gives it (interpolators.py:121-139)."""
        lon = np.asarray(lon, dtype=np.float32)
        lat = np.asarray(lat, dtype=np.float32)
        d = self.desc
        d.nx, d.ny = len(lon), len(lat)
        d.x0, d.xspan = float(lon[0]), float(np.float32(lon[-1] - lon[0]))
        d.y0, d.yspan = float(lat[0]), float(np.float32(lat[-1] - lat[0]))
        self.lon, self.lat = lon, lat
        self.engine.order_after_copies()          # a prefetch into one of the slots may still be in flight on the copy stream
        self.engine._check(self.engine.lib.od_group_set_window(self.engine.ctx, self.gid, C.byref(d)))
        self.resident = [None] * self.n_slots
        self.ready = [None] * self.n_slots

    def set_fallback(self, fallback):
        """environment:fallback:* of this group's variables; read by the kernels at every launch, so that a reader that was
        bound earlier (a direct get_variables_interpolated call, another model instance) follows the current run's values."""
        fb = list(fallback) + [None] * (2 - len(fallback))
        fb = [float('nan') if v is None else float(v) for v in fb]
        self.desc.fallback[0], self.desc.fallback[1] = fb[0], fb[1]
        self.engine._check(self.engine.lib.od_group_set_fallback(self.engine.ctx, self.gid, fb[0], fb[1]))

    def __del__(self):
        try:
            self.engine.free_group(self)
        except Exception:
            pass

    # -- slab residency -------------------------------------------------------------------
    def _victim(self, pinned):
        cand = [s for s in range(self.n_slots) if self.resident[s] not in pinned or self.resident[s] is None]
        if not cand:
            return None
        return min(cand, key=lambda k: (self.resident[k] is not None, self.use[k]))

    def _load(self, ti, s):
        """Bring the slab of time index ti into ring slot s on the engine's CURRENT stream: the rank that reads (every rank when
        the run is not distributed) uploads it from the supplier and fills its NaN holes; in a distributed run the other ranks
        receive it by a broadcast straight into their ring slot (NCCL over NVLink on the GPU box; SURVEY 8(e))."""
        eng = self.engine
        d = eng.dist
        eng.order_after_copies()       # the NaN fill's scratch buffers are per context: never two loads in flight on two streams
        if d is None or d.rank == d.src:
            for c in range(self.ncomp):
                eng.upload(self.gid, s, c, self.supplier(ti, c))
                if self.fill_nan:
                    eng.fill_nan(self.gid, s, c, self.fill_nan)
        if d is not None:
            for c in range(self.ncomp):
                d.broadcast(eng.slot_tensor(self, s, c))
            if d.rank != d.src:
                eng.touch(self.gid, s)
            d.slabs_broadcast += 1

    def slot_of(self, ti, pinned=()):
        """Ring slot holding time index ti, loading it if necessary (never evicting `pinned`)."""
        self._tick += 1
        if ti in self.resident:
            s = self.resident.index(ti)
            self.use[s] = self._tick
            if self.ready[s] is not None:                 # prefetched on the copy stream: order the compute stream behind it
                self.engine.wait_event(self.ready[s])
                self.ready[s] = None
            return s
        s = self._victim(pinned)
        assert s is not None, 'no free ring slot'
        self._load(ti, s)
        self.resident[s] = ti
        self.ready[s] = None
        self.use[s] = self._tick
        return s

    def prefetch(self, ti, pinned=()):
        """Start loading the slab of time index ti into a free ring slot on the engine's COPY stream, so that the upload (and,
        in a distributed run, its broadcast) overlaps the steps that still use the current pair -- the double-buffered block
        supplier of StructuredReader's before / after cache (readers/basereader/structured.py:243-318).  The copy stream
        first waits for the work already queued on the compute stream (kernels that may still read the slot being replaced)."""
        if not self.prefetch_on or ti < 0 or ti >= len(self.times) or ti in self.resident:
            return False
        s = self._victim(pinned)
        if s is None or self.resident[s] in pinned:
            return False
        eng = self.engine
        if not eng.begin_copy_stream():
            return False
        try:
            self._load(ti, s)
            self.ready[s] = eng.end_copy_stream()
        except Exception:
            eng.end_copy_stream()
            raise
        self.resident[s] = ti
        self.use[s] = 0                                   # least recently used until somebody asks for it
        return True

    def sample(self, t, pinned=()):
        """od_time_sample for time t (uploads slabs as needed)."""
        ts = TimeSample()
        br = bracket(self.times, t)
        if br is None:
            ts.mode = OD_T_MISSING
            return ts, ()
        ib, ia, w = br
        if ia is None:
            ts.slot_a = self.slot_of(ib, pinned)
            ts.slot_b = -1
            ts.mode = OD_T_FIRST
            return ts, (ib,)
        sa = self.slot_of(ib, tuple(pinned) + (ia,))
        sb = self.slot_of(ia, tuple(pinned) + (ib,))
        ts.slot_a, ts.slot_b, ts.mode, ts.w = sa, sb, OD_T_LERP, w
        if self.n_slots > 2 and len(self.times) > 2:
            # the slab the run needs next: after the pair in a forward run, before it in a backward run
            nxt = ia + 1 if self.engine.direction >= 0 else ib - 1
            self.prefetch(nxt, tuple(pinned) + (ib, ia))
        return ts, (ib, ia)


def bind_process_to_gpu_numa(device_index):
    """Pin this process (and, by first touch, the pinned host buffers it allocates afterwards) to the CPUs of the NUMA node the
    GPU hangs off: one process per GPU, host staging memory on the GPU's own socket -- otherwise half of the ranks of an 8-GPU
    box push their PCIe traffic through the inter-socket link.  Returns a dict describing what was done (never raises)."""
    import os
    import subprocess
    info = {'device': int(device_index), 'bound': False}
    try:
        bus = subprocess.run(['nvidia-smi', '-i', str(device_index), '--query-gpu=pci.bus_id', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=20).stdout.strip().lower()
        if not bus:
            return info
        if len(bus.split(':')[0]) == 8:          # nvidia-smi prints an 8-digit PCI domain, sysfs uses 4
            bus = bus[4:]
        node_path = '/sys/bus/pci/devices/%s/numa_node' % bus
        node = int(open(node_path).read().strip())
        info['pci_bus_id'], info['numa_node'] = bus, node
        if node < 0:
            return info
        cpus = set()
        for part in open('/sys/devices/system/node/node%d/cpulist' % node).read().strip().split(','):
            a, _, b = part.partition('-')
            cpus.update(range(int(a), int(b or a) + 1))
        cpus &= os.sched_getaffinity(0)
        if cpus:
            os.sched_setaffinity(0, cpus)
            info['bound'], info['cpus'] = True, len(cpus)
    except Exception as ex:
        info['error'] = repr(ex)[:120]
    return info


class DistContext:
    """The torch.distributed job of a sharded run: particle-index shards, replicated forcing (SURVEY 8(e))."""

    def __init__(self, dist, rank, world, src=0, group=None):
        self.dist, self.rank, self.world, self.src, self.group = dist, rank, world, src, group
        self.slabs_broadcast = 0
        self.bcast_group = group
        self.bcast_ctas = None
        # The slab broadcasts run on the copy stream beside the step kernels, one slab ahead of the run.  A rank that reaches its
        # broadcast before the reading rank does keeps the collective's kernel resident -- spinning on the peer -- for as long as
        # that takes, and with NCCL's default budget (up to 32 thread blocks) that kernel takes a fifth of the SMs away from the
        # step kernel (measured at N = 2: 1.14 instead of 0.92 ms per step on the waiting rank).  The broadcasts therefore get a
        # communicator of their own that is limited to a few thread blocks; they have six steps of slack.
        import os
        try:
            ctas = int(os.environ.get('OD_BCAST_CTAS', '4'))
            if ctas > 0 and dist.get_backend(group) == 'nccl':
                import torch
                opts = torch.distributed.ProcessGroupNCCL.Options()
                opts.config.max_ctas = ctas
                opts.config.min_ctas = 1
                ranks = list(range(dist.get_world_size())) if group is None else dist.get_process_group_ranks(group)
                self.bcast_group = dist.new_group(ranks=ranks, backend='nccl', pg_options=opts)
                self.bcast_ctas = ctas
        except Exception:                  # an older torch / NCCL without the option: the job's own communicator
            self.bcast_group = group

    def broadcast(self, tensor):
        self.dist.broadcast(tensor, self.src, group=self.bcast_group)

    def allreduce_bbox(self, eng, bbox):
        """(min, max, min, max) over all ranks; a rank without elements contributes nothing (NaN)."""
        torch = eng.torch
        big = 1e300
        v = [(-bbox[0] if bbox[0] == bbox[0] else -big), (bbox[1] if bbox[1] == bbox[1] else -big),
             (-bbox[2] if bbox[2] == bbox[2] else -big), (bbox[3] if bbox[3] == bbox[3] else -big)]
        t = torch.tensor(v, dtype=torch.float64, device=eng.device)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX, group=self.group)
        r = t.cpu().tolist()
        out = (-r[0], r[1], -r[2], r[3])
        return tuple(float('nan') if abs(x) >= big else x for x in out)

    def shard(self, n_total):
        from .sharding import shard_range
        return shard_range(n_total, self.rank, self.world)


_default = {}


def default_engine(device=None):
    """Process-wide Engine for the current CUDA device (LOCAL_RANK under torchrun)."""
    import os
    if device is None:
        device = int(os.environ.get('LOCAL_RANK', '0'))
    if device not in _default:
        _default[device] = Engine(device)
    return _default[device]


class Engine:
    def __init__(self, device=0):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError('opendrift_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback')
        self.torch = torch
        self.lib = _lib.load()
        self.device = torch.device('cuda', device)
        torch.cuda.set_device(self.device)
        ctx = C.c_void_p()
        rc = self.lib.od_create(device, C.byref(ctx))
        if rc != 0:
            raise RuntimeError('od_create failed (%d)' % rc)
        self.ctx = ctx
        self.use_stream(torch.cuda.current_stream(self.device))
        self.groups = weakref.WeakValueDictionary()     # gid -> FieldGroup (owned by the reader that bound it)
        # arithmetic of the step kernels when a call does not say (include/odcuda.h OD_MATH_*): bit-exact sampling +
        # short-arc series geodesic; MATH_EXACT replays the reference operation by operation, MATH_FAST is float32
        self.math_mode = _lib.OD_MATH_SERIES
        self.dist = None               # DistContext of a distributed run (one process per GPU), else None
        self.direction = 1             # +1 forward run, -1 backward run (which slab to prefetch)
        self._main_stream = torch.cuda.current_stream(self.device)
        self._copy_stream = None
        self._in_copy = False

    # -- streams: compute stream + one copy stream for slab prefetch ----------------------------------------------------
    def wait_event(self, ev):
        self.torch.cuda.current_stream(self.device).wait_event(ev)

    def order_after_copies(self):
        """Make the current stream wait for whatever the copy stream still has queued (no-op while on the copy stream)."""
        ev = getattr(self, '_last_copy_event', None)
        if ev is not None and not self._in_copy:
            self.wait_event(ev)
            self._last_copy_event = None

    def begin_copy_stream(self):
        """Route the library's launches and copies (and torch's, e.g. a broadcast) to the copy stream; False when nested."""
        if self._in_copy:
            return False
        torch = self.torch
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        self._main_stream = torch.cuda.current_stream(self.device)
        self._copy_stream.wait_stream(self._main_stream)       # slots being replaced may still be read by queued kernels
        self._ctx_mgr = torch.cuda.stream(self._copy_stream)
        self._ctx_mgr.__enter__()
        self.use_stream(self._copy_stream)
        self._in_copy = True
        return True

    def end_copy_stream(self):
        """Back to the compute stream; returns an event that marks the end of what was queued on the copy stream."""
        ev = self.torch.cuda.Event()
        ev.record(self._copy_stream)
        self._ctx_mgr.__exit__(None, None, None)
        self.use_stream(self._main_stream)
        self._in_copy = False
        self._last_copy_event = ev
        return ev

    def enable_distributed(self, src=0, group=None):
        """Join the torch.distributed job this process belongs to (torchrun: one process per GPU): forcing slabs are read by
        rank `src` and broadcast into the other ranks' ring slots.  A no-op for a single process."""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            self.dist = DistContext(dist, dist.get_rank(group), dist.get_world_size(group), src, group)
        return self.dist

    def touch(self, gid, slot):
        self._check(self.lib.od_group_touch(self.ctx, gid, slot))

    def close(self):
        if getattr(self, 'ctx', None):
            self.lib.od_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError('libodcuda: %s (status %d)' % (self.lib.od_last_error(self.ctx).decode(), rc))

    def use_stream(self, stream):
        self._check(self.lib.od_set_stream(self.ctx, C.c_void_p(stream.cuda_stream)))

    def set_tile(self, on):
        """TMA-staged field boxes in shared memory for the RK kernels (cell-sorted particle arrays)."""
        self._check(self.lib.od_set_option(self.ctx, _lib.OD_OPT_TILE, 1 if on else 0))

    def set_spec(self, on):
        """The specialised RK4 step kernel for launches that qualify (csrc/od_spec.cuh; on by default, results are
        bit-identical either way)."""
        self._check(self.lib.od_set_option(self.ctx, _lib.OD_OPT_SPEC, 1 if on else 0))

    def sync(self):
        self._check(self.lib.od_sync(self.ctx))

    def launches(self):
        return int(self.lib.od_launch_count(self.ctx))

    # -- buffers --------------------------------------------------------------------------
    def to_device(self, a, dtype=None):
        t = self.torch.as_tensor(np.ascontiguousarray(a))
        if dtype is not None:
            t = t.to(dtype)
        return t.to(self.device, non_blocking=True)

    def empty(self, n, dtype):
        return self.torch.empty(n, dtype=dtype, device=self.device)

    # -- groups ---------------------------------------------------------------------------
    def add_group(self, lon, lat, z, ncomp, times, supplier, fallback, n_slots=3, names=None, **proj_kw):
        free = [k for k in range(_lib.OD_MAX_GROUPS) if k not in self.groups]
        if not free:
            gc.collect()
            free = [k for k in range(_lib.OD_MAX_GROUPS) if k not in self.groups]
        if not free:
            raise RuntimeError('all %d field groups of this engine are in use; release readers you no longer need'
                               % _lib.OD_MAX_GROUPS)
        gid = free[0]
        g = FieldGroup(self, gid, lon, lat, z, ncomp, times, supplier, fallback, n_slots, names, **proj_kw)
        self.groups[gid] = g
        return g

    def free_group(self, group):
        """Release a group's device slabs (its id becomes reusable)."""
        if self.ctx and self.groups.get(group.gid) in (group, None) and not group.freed:
            group.freed = True
            self._check(self.lib.od_group_free(self.ctx, group.gid))
            self.groups.pop(group.gid, None)

    def upload(self, gid, slot, comp, data):
        torch = self.torch
        if isinstance(data, torch.Tensor):
            assert data.dtype == torch.float32 and data.is_contiguous()
            on_dev = 1 if data.is_cuda else 0
            self._check(self.lib.od_group_upload(self.ctx, gid, slot, comp, C.c_void_p(data.data_ptr()), on_dev))
            if not on_dev and not data.is_pinned():
                self.sync()          # pageable host memory may be reused by the caller; pinned slabs are the caller's to keep
        else:
            a = np.ascontiguousarray(data, dtype=np.float32)
            self._check(self.lib.od_group_upload(self.ctx, gid, slot, comp, a.ctypes.data_as(C.c_void_p), 0))
            self.sync()

    def fill_nan(self, gid, slot, comp, iterations=10, report=False):
        """linearNDFast NaN fill of an uploaded slab (asynchronous unless report=True)."""
        if report:
            rem = C.c_int64()
            self._check(self.lib.od_group_fill_nan(self.ctx, gid, slot, comp, iterations, C.byref(rem)))
            return int(rem.value)
        self._check(self.lib.od_group_fill_nan(self.ctx, gid, slot, comp, iterations, None))

    def slot_tensor(self, group, slot, comp):
        """The ring slot as a CUDA tensor (e.g. the target of a torch.distributed broadcast)."""
        p = C.c_void_p()
        self._check(self.lib.od_group_slot_ptr(self.ctx, group.gid, slot, comp, C.byref(p)))
        d = group.desc
        n = d.nx * d.ny * d.nz
        # wrap the raw pointer without copying
        iface = {'shape': (n,), 'typestr': '<f4', 'data': (p.value, False), 'version': 3}

        class _W:
            __cuda_array_interface__ = iface
        return self.torch.as_tensor(_W(), device=self.device)

    # -- kernels --------------------------------------------------------------------------
    def interp(self, group, t, lon, lat, z=None, pos_f32=False, raw=False, rotate=True, out_f64=False, nearest=False):
        """get_variables_interpolated fast path on device tensors -> list of float32 tensors (float64 with out_f64: the reader's
        own precision, raw only).  nearest: the nearest grid point, as the reference samples land_binary_mask."""
        n = lon.numel()
        ts, _ = group.sample(t)
        outs = [self.empty(n, self.torch.float64 if out_f64 else self.torch.float32) for _ in range(group.ncomp)]
        self._check(self.lib.od_interp(self.ctx, group.gid, C.byref(ts), n, _ptr(lon), _ptr(lat), _ptr(z),
                                       (1 if pos_f32 else 0) | (2 if raw else 0) | (4 if (z is not None and z.dtype == self.torch.float64) else 0)
                                       | (0 if rotate else 8) | (_lib.OD_INTERP_OUT_F64 if out_f64 else 0) | (_lib.OD_INTERP_NEAREST if nearest else 0),
                                       _ptr(outs[0]), _ptr(outs[1]) if group.ncomp == 2 else None))
        return outs

    def coastline(self, mask, lon, lat, z, age, status, moving, ids, prev_lon, prev_lat, id_base, action, stranded_code=0,
                  seeded_code=0, missing_code=0, check_seeded=False, ssh=0.0):
        """interact_with_coastline (basemodel/__init__.py:671-746) for a sampled land_binary_mask; returns the counts
        (stranded, seeded_on_land, missing_data, moved back)."""
        a = _lib.CoastArgs()
        a.n = lon.numel()
        a.d_mask, a.d_lon, a.d_lat, a.d_z, a.d_age = _ptr(mask), _ptr(lon), _ptr(lat), _ptr(z), _ptr(age)
        a.d_status, a.d_moving, a.d_ids = _ptr(status), _ptr(moving), _ptr(ids)
        a.d_prev_lon, a.d_prev_lat = _ptr(prev_lon), _ptr(prev_lat)
        a.n_total = 0 if prev_lon is None else prev_lon.numel()
        a.id_base, a.action = int(id_base), {'stranding': 1, 'previous': 2, 'seafloor_previous': 3}[action]
        a.ssh = float(ssh)
        a.stranded_code, a.seeded_code, a.missing_code = int(stranded_code), int(seeded_code), int(missing_code)
        a.check_seeded = 1 if check_seeded else 0
        a.z_f64 = 1 if (z is not None and z.dtype == self.torch.float64) else 0
        a.age_f64 = 1 if (age is not None and age.dtype == self.torch.float64) else 0
        counts = (C.c_int64 * 4)()
        a.h_counts = C.cast(counts, C.POINTER(C.c_int64))
        self._check(self.lib.od_coastline(self.ctx, C.byref(a)))
        return tuple(int(c) for c in counts)

    def store_previous(self, lon, lat, ids, id_base, prev_lon, prev_lat):
        """update_previous_state (:642-669) for lon / lat: previous[ID - id_base] = the present position (float32)."""
        self._check(self.lib.od_store_previous(self.ctx, lon.numel(), _ptr(lon), _ptr(lat), _ptr(ids), int(id_base), prev_lon.numel(),
                                               _ptr(prev_lon), _ptr(prev_lat)))

    def store_previous_env(self, present, ids, age, dt, id_base, store):
        """update_previous_state (:642-657) for one float32 environment variable: returns the previous values of the active
        elements and stores the present ones into `store` ([n_total] float32, keyed by ID - id_base).  age: age_seconds
        on a step that released elements, else None."""
        torch = self.torch
        assert present.dtype == torch.float32 and ids.dtype == torch.int32 and store.dtype == torch.float32
        prev = self.empty(present.numel(), torch.float32)
        age_f64 = 0
        if age is not None:
            assert age.dtype in (torch.float32, torch.float64)
            age_f64 = 1 if age.dtype == torch.float64 else 0
        self._check(self.lib.od_store_previous_env(self.ctx, present.numel(), _ptr(present), _ptr(ids), _ptr(age), age_f64, float(dt),
                                                   int(id_base), store.numel(), _ptr(store), _ptr(prev)))
        return prev

    def vertical_advection_corrected(self, z, w, ssh, ssh_prev, floor, moving, at_surface, dt):
        """OceanDrift.vertical_advection with drift:vertical_advection_correction (oceandrift.py:325-350), in place on z.
        floor: float32 tensor or a number."""
        torch = self.torch
        assert z.dtype in (torch.float32, torch.float64) and moving.dtype == torch.int32
        assert w.dtype == ssh.dtype == ssh_prev.dtype == torch.float32
        fl, fc = (floor, 0.0) if hasattr(floor, 'data_ptr') else (None, float(floor))
        assert fl is None or fl.dtype == torch.float32
        self._check(self.lib.od_vertical_advection_corrected(self.ctx, z.numel(), _ptr(z), 1 if z.dtype == torch.float64 else 0, _ptr(w),
                                                             _ptr(ssh), _ptr(ssh_prev), _ptr(fl), fc, _ptr(moving),
                                                             1 if at_surface else 0, float(dt)))

    def geod_fwd(self, lon, lat, az, dist):
        self._check(self.lib.od_geod_fwd(self.ctx, lon.numel(), _ptr(lon), _ptr(lat), _ptr(az), _ptr(dist)))

    def update_positions(self, lon, lat, xvel, yvel, moving, dt):
        f64 = 1 if xvel.dtype == self.torch.float64 else 0
        assert xvel.dtype == yvel.dtype
        self._check(self.lib.od_update_positions(self.ctx, lon.numel(), _ptr(lon), _ptr(lat), _ptr(xvel),
                                                 _ptr(yvel), f64, _ptr(moving), float(dt)))

    def _advect_args(self, a, group, scheme, t, dt_seconds, half, full, lon, lat, z, factor, moving,
                     k1=None, truncate_below=None, env_out=None, pos_f32=False, fast=None, noise=None, noise_kinds=0, chain=()):
        a.scheme = SCHEMES[scheme] if isinstance(scheme, str) else scheme
        if noise is not None:
            a.d_noise_cur, a.noise_kinds = noise.data_ptr(), int(noise_kinds)
        a.fast = self.math_mode if fast is None else int(fast)      # OD_MATH_EXACT 0 / FAST 1 (True) / SERIES 2
        a.pos_f32 = 1 if pos_f32 else 0
        a.group_uv = group.gid
        pinned = ()
        if k1 is None:
            a.t_start, p = group.sample(t)
            pinned += p
        if a.scheme != _lib.OD_EULER:
            a.t_mid, p = group.sample(half, pinned)
            pinned += p
        if a.scheme == _lib.OD_RK4:
            a.t_end, p = group.sample(full, pinned)
        # further current groups in reader priority order (sampled where the ones before them give NaN)
        if len(chain) > _lib.OD_MAX_CHAIN:
            raise ValueError('at most %d chained current readers' % _lib.OD_MAX_CHAIN)
        a.n_chain = len(chain)
        for k, cg in enumerate(chain):
            a.chain_group[k] = cg.gid
            held = ()                      # slabs the earlier samples of this group refer to must stay in their ring slots
            if k1 is None:
                a.chain_t[k][0], q = cg.sample(t)
                held += q
            if a.scheme != _lib.OD_EULER:
                a.chain_t[k][1], q = cg.sample(half, held)
                held += q
            if a.scheme == _lib.OD_RK4:
                a.chain_t[k][2], q = cg.sample(full, held)
        a.dt = float(dt_seconds)
        a.n = lon.numel()
        a.d_lon, a.d_lat = lon.data_ptr(), lat.data_ptr()
        a.d_z = z.data_ptr() if z is not None else None
        a.z_f64 = 1 if (z is not None and z.dtype == self.torch.float64) else 0
        if factor is not None:
            a.d_factor = factor.data_ptr()
            a.factor_f64 = 1 if factor.dtype == self.torch.float64 else 0
        else:
            a.factor_f64 = 1
        a.d_moving = moving.data_ptr() if moving is not None else None
        if k1 is not None:
            a.d_k1_u, a.d_k1_v = k1[0].data_ptr(), k1[1].data_ptr()
        a.truncate_below = float(truncate_below) if truncate_below else 0.0
        if env_out is not None:
            a.d_env_u, a.d_env_v = env_out[0].data_ptr(), env_out[1].data_ptr()

    def advect_current(self, group, scheme, t, dt, lon, lat, z=None, factor=None, moving=None, k1=None,
                       truncate_below=None, env_out=None, pos_f32=False, fast=None, noise=None, noise_kinds=0, chain=()):
        """advect_ocean_current on device tensors (in place).  t is the reader-time object (datetime
        or seconds), dt a timedelta-like or seconds."""
        dts = dt.total_seconds() if hasattr(dt, 'total_seconds') else float(dt)
        a = AdvectArgs()
        self._advect_args(a, group, scheme, t, dts, t + dt / 2, t + dt, lon, lat, z, factor, moving, k1,
                          truncate_below, env_out, pos_f32, fast, noise, noise_kinds, chain)
        self._check(self.lib.od_advect_current(self.ctx, C.byref(a)))

    # -- analytical reader on a projected plane (od_analytic_*) ----------------------------------------------
    def analytic_interp(self, desc, t_seconds, lon, lat, pos_f32=False):
        """Reader chain of an analytical projected reader on device tensors -> (u, v) float32, NaN where uncovered."""
        n = lon.numel()
        u, v = self.empty(n, self.torch.float32), self.empty(n, self.torch.float32)
        self._check(self.lib.od_analytic_interp(self.ctx, C.byref(desc), float(t_seconds), n, _ptr(lon), _ptr(lat),
                                                1 if pos_f32 else 0, _ptr(u), _ptr(v)))
        return u, v

    def analytic_advect(self, desc, scheme, t_seconds, dt_seconds, lon, lat, factor=None, moving=None, k1=None,
                        env_out=None, pos_f32=False, fast=None):
        """advect_ocean_current with an analytical reader as the current (in place).  t_seconds = (t, t + dt/2, t + dt)
        in seconds since the reader's initial_time."""
        a = _lib.AnalyticAdvectArgs()
        a.scheme = SCHEMES[scheme] if isinstance(scheme, str) else scheme
        a.math = self.math_mode if fast is None else int(fast)
        a.pos_f32 = 1 if pos_f32 else 0
        a.t_start, a.t_mid, a.t_end = (float(x) for x in t_seconds)
        a.dt = float(dt_seconds)
        a.n = lon.numel()
        a.d_lon, a.d_lat = lon.data_ptr(), lat.data_ptr()
        if factor is not None:
            a.d_factor = factor.data_ptr()
            a.factor_f64 = 1 if factor.dtype == self.torch.float64 else 0
        else:
            a.factor_f64 = 1
        a.d_moving = moving.data_ptr() if moving is not None else None
        if k1 is not None:
            a.d_k1_u, a.d_k1_v = k1[0].data_ptr(), k1[1].data_ptr()
        if env_out is not None:
            a.d_env_u, a.d_env_v = env_out[0].data_ptr(), env_out[1].data_ptr()
        self._check(self.lib.od_analytic_advect(self.ctx, C.byref(desc), C.byref(a)))

    # -- output buffer on the device (od_history_scatter) ------------------------------------------------------
    def history_scatter(self, ids, lon, lat, z, status, bufs, col):
        """state_to_buffer: scatter lon / lat / z / status of the active elements into column `col` of the
        [n_total, ncols] device buffers bufs = (lon f32, lat f32, z f32, status i32), rows addressed by element ID."""
        torch = self.torch
        a = _lib.HistoryArgs()
        a.n, a.n_total, a.col, a.ncols = ids.numel(), bufs[0].shape[0], int(col), bufs[0].shape[1]
        assert ids.dtype == torch.int32 and status.dtype == torch.int32 and lon.dtype == torch.float64 and lat.dtype == torch.float64
        assert z.dtype in (torch.float32, torch.float64) and all(b.is_contiguous() for b in bufs)
        a.z_f64 = 1 if z.dtype == torch.float64 else 0
        a.d_ids, a.d_lon, a.d_lat, a.d_z, a.d_status = ids.data_ptr(), lon.data_ptr(), lat.data_ptr(), z.data_ptr(), status.data_ptr()
        a.d_buf_lon, a.d_buf_lat, a.d_buf_z, a.d_buf_status = (b.data_ptr() for b in bufs)
        self._check(self.lib.od_history_scatter(self.ctx, C.byref(a)))

    def bookkeeping(self, lon, lat, z, age, status, moving, ids, dt_age, max_age=None, domain=None, outside_code=0,
                    retired_code=0, pos_f32=False, buf=None, only_deactivated=False, counts=True, id_base=0):
        """deactivate_outside + state_to_buffer + increase_age_and_retire in one pass (od_bookkeeping).  buf: the four
        [n_total] float32 / float32 / float32 / int32 device tensors of the output column to fill (or None).
        Returns (newly outside, newly retired, elements with status != 0) when counts (synchronises), else None."""
        torch = self.torch
        a = _lib.BookkeepArgs()
        a.n = lon.numel()
        assert lon.dtype == torch.float64 and lat.dtype == torch.float64 and status.dtype == torch.int32 and moving.dtype == torch.int32
        assert age.dtype in (torch.float32, torch.float64)
        a.d_lon, a.d_lat, a.d_age, a.d_status, a.d_moving = lon.data_ptr(), lat.data_ptr(), age.data_ptr(), status.data_ptr(), moving.data_ptr()
        a.age_f64 = 1 if age.dtype == torch.float64 else 0
        a.dt_age = float(dt_age)
        a.max_age = float('nan') if max_age is None else float(max_age)
        W, E, S, N = domain if domain is not None else (None, None, None, None)
        a.west, a.east, a.south, a.north = (float('nan') if v is None else float(v) for v in (W, E, S, N))
        a.outside_code, a.retired_code = int(outside_code), int(retired_code)
        a.pos_f32 = 1 if pos_f32 else 0
        a.only_deactivated = 1 if only_deactivated else 0
        if buf is not None:
            assert ids.dtype == torch.int32 and z.dtype in (torch.float32, torch.float64)
            a.d_ids, a.d_z, a.z_f64 = ids.data_ptr(), z.data_ptr(), 1 if z.dtype == torch.float64 else 0
            # rows are addressed by element ID; a shard of a distributed run holds the IDs id_base .. id_base + rows - 1
            a.n_total, a.col, a.ncols = buf[0].numel() + int(id_base), 0, 1
            a.d_buf_lon, a.d_buf_lat, a.d_buf_z, a.d_buf_status = (b.data_ptr() - 4 * int(id_base) for b in buf)
        c = (C.c_int64 * 3)()
        if counts:
            a.h_counts = c
        self._check(self.lib.od_bookkeeping(self.ctx, C.byref(a)))
        return (int(c[0]), int(c[1]), int(c[2])) if counts else None

    def vertical_buoyancy(self, z_in, z_out, terminal_velocity, dt, sea_floor=None, sea_surface_height=0.0, status=None, moving=None,
                          seafloor_code=0, count=False):
        """OceanDrift.vertical_buoyancy / interact_with_seafloor on device tensors (od_vertical_buoyancy); z_out may be z_in."""
        torch = self.torch
        a = _lib.BuoyancyArgs()
        a.n = z_in.numel()
        assert z_in.dtype == z_out.dtype and z_in.dtype in (torch.float32, torch.float64)
        a.d_z_in, a.d_z_out, a.z_f64 = z_in.data_ptr(), z_out.data_ptr(), 1 if z_in.dtype == torch.float64 else 0
        if terminal_velocity is not None:
            assert terminal_velocity.dtype in (torch.float32, torch.float64)
            a.d_terminal_velocity, a.tv_f64 = terminal_velocity.data_ptr(), 1 if terminal_velocity.dtype == torch.float64 else 0
        if sea_floor is not None:
            assert sea_floor.dtype == torch.float32
            a.d_sea_floor = sea_floor.data_ptr()
        a.dt, a.sea_surface_height, a.seafloor_code = float(dt), float(sea_surface_height), int(seafloor_code)
        if status is not None:
            assert status.dtype == torch.int32 and moving.dtype == torch.int32
            a.d_status, a.d_moving = status.data_ptr(), moving.data_ptr()
        c = C.c_int64(0)
        if count:
            a.h_n_deactivated = C.pointer(c)
        self._check(self.lib.od_vertical_buoyancy(self.ctx, C.byref(a)))
        return int(c.value) if count else None

    def _step_args(self, s, group, scheme, t, dts, dt, lon, lat, z, factor, moving, truncate_below, wind, wdf,
                   wind_drift_depth, w_group, w_at_surface, rand, diffusivity, pos_f32, z_update, fast, noise, noise_kinds,
                   wind_noise, chain=()):
        self._advect_args(s.cur, group, scheme, t, dts, t + dt / 2, t + dt, lon, lat, z, factor, moving,
                          None, truncate_below, None, pos_f32, fast, noise, noise_kinds, chain)
        s.group_wind = -1
        s.group_w = -1
        if wind is not None:
            s.group_wind = wind.gid
            s.t_wind, _ = wind.sample(t)
            s.d_wdf = wdf.data_ptr()
            s.wdf_f64 = 1 if wdf.dtype == self.torch.float64 else 0
            s.wind_drift_depth = float(wind_drift_depth)
            if wind_noise is not None:
                s.d_noise_wind = wind_noise.data_ptr()
        if w_group is not None:
            s.group_w = w_group.gid
            s.t_w, _ = w_group.sample(t)
            s.w_at_surface = 1 if w_at_surface else 0
            zu = z if z_update is None else z_update
            s.d_z_inout = zu.data_ptr()
            s.z_inout_f64 = 1 if zu.dtype == self.torch.float64 else 0
        if rand is not None:
            s.d_rand_x, s.d_rand_y = rand[0].data_ptr(), rand[1].data_ptr()
            if hasattr(diffusivity, 'data_ptr'):
                s.d_diffusivity = diffusivity.data_ptr()
            else:
                s.diffusivity_const = float(diffusivity)

    def step_oceandrift(self, group, scheme, t, dt, lon, lat, z=None, factor=None, moving=None,
                        truncate_below=None, wind=None, wdf=None, wind_drift_depth=0.1, w_group=None,
                        w_at_surface=False, rand=None, diffusivity=None, pos_f32=False, z_update=None, fast=None, noise=None, noise_kinds=0,
                        wind_noise=None, chain=()):
        """One fused OceanDrift step.  z is the depth used for sampling; z_update (default: z itself) is the depth
        array that vertical advection updates -- a different buffer after vertical mixing.  chain: further current groups
        in reader priority order."""
        dts = dt.total_seconds() if hasattr(dt, 'total_seconds') else float(dt)
        s = StepArgs()
        self._step_args(s, group, scheme, t, dts, dt, lon, lat, z, factor, moving, truncate_below, wind, wdf, wind_drift_depth,
                        w_group, w_at_surface, rand, diffusivity, pos_f32, z_update, fast, noise, noise_kinds, wind_noise, chain)
        self._check(self.lib.od_step_oceandrift(self.ctx, C.byref(s)))

    @staticmethod
    def _host_ptr(x, dtypes):
        if x is None:
            return None, None
        if isinstance(x, np.ndarray):
            assert x.dtype in [np.dtype(d) for d in dtypes] and x.flags['C_CONTIGUOUS']
            return x.ctypes.data, x.dtype.itemsize
        assert not x.is_cuda and x.is_contiguous() and x.element_size() in [np.dtype(d).itemsize for d in dtypes]
        return x.data_ptr(), x.element_size()

    def _host_io(self, h_lon, h_lat, h_z, h_out_lon, h_out_lat, h_out_z, chunks):
        io = _lib.HostIO()
        io.h_lon, _ = self._host_ptr(h_lon, ['f8'])
        io.h_lat, _ = self._host_ptr(h_lat, ['f8'])
        io.h_z, zsz = self._host_ptr(h_z, ['f4', 'f8'])
        io.h_out_lon, _ = self._host_ptr(h_lon if h_out_lon is None else h_out_lon, ['f8'])
        io.h_out_lat, _ = self._host_ptr(h_lat if h_out_lat is None else h_out_lat, ['f8'])
        io.h_out_z, zo = self._host_ptr(h_z if h_out_z is None else h_out_z, ['f4', 'f8'])
        assert zo == zsz
        io.chunks = int(chunks)
        torch = self.torch
        if not hasattr(self, '_host_dummy'):
            self._host_dummy = (self.empty(1, torch.float64), self.empty(1, torch.float64), self.empty(1, torch.float32),
                                self.empty(1, torch.float64))
        dz = None if h_z is None else (self._host_dummy[3] if zsz == 8 else self._host_dummy[2])
        return io, dz

    def step_oceandrift_host(self, group, scheme, t, dt, h_lon, h_lat, h_z=None, h_out_lon=None, h_out_lat=None, h_out_z=None,
                             factor=None, moving=None, truncate_below=None, wind=None, wdf=None, wind_drift_depth=0.1,
                             w_group=None, w_at_surface=False, rand=None, diffusivity=None, chunks=0, pos_f32=False, fast=None):
        """The fused OceanDrift step for HOST arrays (od_step_oceandrift_host): positions and depths in, positions (and
        depths, when vertical advection is on) out, pipelined in chunks like advect_current_host."""
        io, dz = self._host_io(h_lon, h_lat, h_z, h_out_lon, h_out_lat, h_out_z, chunks)
        dts = dt.total_seconds() if hasattr(dt, 'total_seconds') else float(dt)
        s = StepArgs()
        self._step_args(s, group, scheme, t, dts, dt, self._host_dummy[0], self._host_dummy[1], dz, factor, moving,
                        truncate_below, wind, wdf, wind_drift_depth, w_group, w_at_surface, rand, diffusivity, pos_f32, None,
                        fast, None, 0, None)
        s.cur.n = int(h_lon.shape[0])
        self._check(self.lib.od_step_oceandrift_host(self.ctx, C.byref(s), C.byref(io)))

    def advect_current_host(self, group, scheme, t, dt, h_lon, h_lat, h_z=None, h_out_lon=None, h_out_lat=None,
                            factor=None, moving=None, chunks=0, pos_f32=False, fast=None):
        """advect_ocean_current for HOST arrays (float64 lon / lat, float32 or float64 z; NumPy arrays or CPU torch
        tensors, pinned for full speed): od_advect_current_host cuts the particle range into chunks whose
        host->device copy, kernel and device->host copy are pipelined on three CUDA streams, so that the PCIe
        transfers of neighbouring chunks overlap each other and the kernel.  Results land in h_out_lon / h_out_lat
        (default: in place).  Returns after everything has completed."""
        io, dz = self._host_io(h_lon, h_lat, h_z, h_out_lon, h_out_lat, None, chunks)
        dts = dt.total_seconds() if hasattr(dt, 'total_seconds') else float(dt)
        a = AdvectArgs()
        self._advect_args(a, group, scheme, t, dts, t + dt / 2, t + dt, self._host_dummy[0], self._host_dummy[1], dz,
                          factor, moving, None, None, None, pos_f32, fast)
        a.n = int(h_lon.shape[0])
        self._check(self.lib.od_advect_current_host(self.ctx, C.byref(a), C.byref(io)))

    def leeway_step(self, wind, cur, t, dt, lon, lat, el, moving=None, status=None, ids=None, rand=None, seed=0,
                    step_index=0, capsize_fraction=0.4, missing_code=1, pos_f32=False, capsizing=None, rand_capsize=None,
                    noise_cur=None, noise_kinds=0, noise_wind=None):
        """Leeway.update on device tensors; el: dict of the per-element coefficient tensors."""
        torch = self.torch
        a = LeewayArgs()
        a.group_wind, a.group_cur = wind.gid, cur.gid
        a.t_wind, _ = wind.sample(t)
        a.t_cur, _ = cur.sample(t)
        a.n = lon.numel()
        a.d_lon, a.d_lat = lon.data_ptr(), lat.data_ptr()
        for k in ('dw_slope', 'dw_offset', 'dw_eps', 'cw_slope', 'cw_offset', 'cw_eps'):
            assert el[k].dtype == torch.float32
            setattr(a, 'd_' + k, el[k].data_ptr())
        assert el['orientation'].dtype == torch.uint8
        a.d_orientation = el['orientation'].data_ptr()
        if el.get('capsized') is not None:
            assert el['capsized'].dtype == torch.uint8
            a.d_capsized = el['capsized'].data_ptr()
        jp = el['jibe_probability']
        a.d_jibe_probability, a.jp_f64 = jp.data_ptr(), 1 if jp.dtype == torch.float64 else 0
        a.d_moving = moving.data_ptr() if moving is not None else None
        a.d_status = status.data_ptr() if status is not None else None
        a.d_ids = ids.data_ptr() if ids is not None else None
        a.d_rand = rand.data_ptr() if rand is not None else None
        a.dt = dt.total_seconds() if hasattr(dt, 'total_seconds') else float(dt)
        a.seed, a.step_index, a.capsize_fraction = int(seed), int(step_index), float(capsize_fraction)
        a.missing_code, a.pos_f32 = int(missing_code), 1 if pos_f32 else 0
        if noise_cur is not None:      # the step's uncertainty draws: float64 [kind][component][n] / [component][n]
            a.d_noise_cur, a.noise_kinds = noise_cur.data_ptr(), int(noise_kinds)
        if noise_wind is not None:
            a.d_noise_wind = noise_wind.data_ptr()
        if capsizing is not None:        # processes:capsizing: (wind_threshold, wind_threshold_sigma); el['capsized'] is updated in place
            assert el.get('capsized') is not None
            a.capsize_on, a.capsize_from = 1, (0 if a.dt >= 0 else 1)
            a.wind_threshold, a.wind_sigma = float(capsizing[0]), float(capsizing[1])
            a.d_rand_capsize = rand_capsize.data_ptr() if rand_capsize is not None else None
        self._check(self.lib.od_leeway_step(self.ctx, C.byref(a)))

    def bbox(self, lon, lat):
        """(lon min, lon max, lat min, lat max) of float64 device tensors, NaNs ignored (synchronises)."""
        out = (C.c_double * 4)()
        self._check(self.lib.od_bbox(self.ctx, lon.numel(), _ptr(lon), _ptr(lat), out))
        return tuple(out)

    def minmax(self, a, b=None):
        """(min, max) of a (+ b) over a float32 device tensor, NaNs ignored (synchronises)."""
        lo, hi = C.c_float(), C.c_float()
        self._check(self.lib.od_minmax_f32(self.ctx, a.numel(), _ptr(a), _ptr(b), C.byref(lo), C.byref(hi)))
        return lo.value, hi.value

    PROFILES = {'monochromatic': 0, 'exponential': 1, 'Phillips': 2, 'windsea_swell': 3}

    def stokes_drift(self, lon, lat, z, us, vs, hs, xwind, ywind, moving, dt, hs_mode, profile, factor=1, windsea_swell=None):
        """factor: Python scalar or a float32 / float64 device tensor; windsea_swell: the six float32 tensors (swell direction,
        period, height, wind-sea direction, period, height) of the combined profile."""
        a = StokesArgs()
        a.factor = 1.0
        if hasattr(factor, 'data_ptr'):
            assert factor.dtype in (self.torch.float32, self.torch.float64)
            a.d_factor, a.factor_f64 = factor.data_ptr(), 1 if factor.dtype == self.torch.float64 else 0
        else:
            a.factor = float(factor)
        if windsea_swell is not None:
            assert all(t.dtype == self.torch.float32 for t in windsea_swell)
            (a.d_swell_dir, a.d_swell_period, a.d_swell_hs, a.d_windsea_dir, a.d_windsea_period,
             a.d_windsea_hs) = (t.data_ptr() for t in windsea_swell)
        a.n = lon.numel()
        a.d_lon, a.d_lat, a.d_z = lon.data_ptr(), lat.data_ptr(), z.data_ptr()
        a.z_f64 = 1 if z.dtype == self.torch.float64 else 0
        a.d_us, a.d_vs = us.data_ptr(), vs.data_ptr()
        a.d_hs = hs.data_ptr() if hs is not None else None
        a.d_xwind = xwind.data_ptr() if xwind is not None else None
        a.d_ywind = ywind.data_ptr() if ywind is not None else None
        a.d_moving = moving.data_ptr() if moving is not None else None
        a.dt, a.hs_mode, a.profile = float(dt), int(hs_mode), self.PROFILES[profile]
        self._check(self.lib.od_stokes_drift(self.ctx, C.byref(a)))

    MIX_MODELS = {'environment': _lib.OD_MIX_ENVIRONMENT, 'windspeed_Large1994': _lib.OD_MIX_LARGE1994,
                  'windspeed_Sundby1983': _lib.OD_MIX_SUNDBY1983, 'constant': _lib.OD_MIX_CONSTANT}

    def vertical_mixing(self, group, t, lon, lat, z_in, dt_mix, ntimes, moving=None, terminal_velocity=None, ids=None,
                        rand=None, seed=0, step_index=0, sea_floor=10000.0, mix_at_surface=False, pos_f32=False,
                        model='environment', wind_speed=None, mld=50.0, background=1.2e-5, k_const=0.0, seafloor_action=0,
                        status=None, seafloor_code=0, iter0=0, skip_surface_stick=False):
        """OceanDrift.vertical_mixing on device tensors; returns the new depth (float64 tensor).
        model 'environment' takes the diffusivity column from `group`; 'windspeed_Large1994' / 'windspeed_Sundby1983' /
        'constant' build it analytically on 1 m levels from wind_speed (float32 tensor) and the mixed layer depth mld
        (float32 tensor or scalar), as oceandrift.py:429-453 does when no ocean-model diffusivity is available."""
        torch = self.torch
        n = lon.numel()
        z_out = self.empty(n, torch.float64)
        a = MixArgs()
        a.ntimes = int(ntimes)
        a.model = self.MIX_MODELS[model]
        if a.model == _lib.OD_MIX_ENVIRONMENT:
            a.group_k = group.gid
            a.t_k, _ = group.sample(t)
        else:
            a.group_k = -1
            if hasattr(mld, 'data_ptr'):
                assert mld.dtype == torch.float32
                a.d_mld = mld.data_ptr()
                mld_max = float(self.minmax(mld)[1])
            else:
                a.mld_const = float(np.float32(mld))
                mld_max = float(np.float32(mld))
            a.nlev = len(np.arange(0, np.float32(mld_max) + 2))          # mixing_z = -np.arange(0, MLD.max() + 2)
            if wind_speed is not None:
                assert wind_speed.dtype == torch.float32
                a.d_wind_speed = wind_speed.data_ptr()
            a.background, a.k_const = float(background), float(k_const)
        a.n = n
        a.d_lon, a.d_lat = lon.data_ptr(), lat.data_ptr()
        a.d_z_in, a.z_in_f64 = z_in.data_ptr(), 1 if z_in.dtype == torch.float64 else 0
        a.d_z_out = z_out.data_ptr()
        a.d_moving = moving.data_ptr() if moving is not None else None
        if terminal_velocity is not None:
            a.d_terminal_velocity = terminal_velocity.data_ptr()
            a.tv_f64 = 1 if terminal_velocity.dtype == torch.float64 else 0
        a.d_ids = ids.data_ptr() if ids is not None else None
        a.d_rand = rand.data_ptr() if rand is not None else None
        if hasattr(sea_floor, 'data_ptr'):
            a.d_sea_floor = sea_floor.data_ptr()
        else:
            a.sea_floor_const = float(sea_floor)
        a.dt_mix, a.seed, a.step_index = float(dt_mix), int(seed), int(step_index)
        a.mix_at_surface, a.pos_f32 = (1 if mix_at_surface else 0), (1 if pos_f32 else 0)
        a.iter0, a.skip_surface_stick = int(iter0), 1 if skip_surface_stick else 0
        a.seafloor_action = int(seafloor_action)          # 'stick to bottom' with a sea-floor reader: 1 lift, 2 deactivate
        nd = C.c_int64(0)
        if a.seafloor_action == 2:
            assert status is not None and moving is not None and status.dtype == torch.int32
            a.d_status, a.d_moving_out, a.seafloor_code = status.data_ptr(), moving.data_ptr(), int(seafloor_code)
            a.h_n_deactivated = C.pointer(nd)
        self._check(self.lib.od_vertical_mixing(self.ctx, C.byref(a)))
        self.last_mix_deactivated = int(nd.value)
        return z_out

    # -- particle exchange of the spatial-tile mode (od_pack_by_owner / od_unpack_records) --------------------------------------
    def pack_by_owner(self, lon, bounds, columns, want_perm=False):
        """Group the elements by the longitude strip that owns them and pack them as records (one row per element, the
        columns side by side).  columns: dict name -> 1-D device tensor (n elements).  Returns (records uint8 [n, rec_bytes],
        counts per owner, layout, perm or None); layout = [(name, dtype, bytes), ...] for unpack_records."""
        torch = self.torch
        n = lon.numel()
        assert lon.dtype == torch.float64 and len(columns) <= _lib.OD_PACK_MAX_COLS and len(bounds) - 1 <= _lib.OD_PACK_MAX_WORLD
        a = _lib.PackArgs()
        a.n, a.d_lon, a.world, a.ncols = n, lon.data_ptr(), len(bounds) - 1, len(columns)
        hb = (C.c_double * len(bounds))(*[float(b) for b in bounds])
        a.h_bounds = hb
        layout, rec = [], 0
        for k, (name, t) in enumerate(columns.items()):
            assert t.is_contiguous() and t.dim() == 1 and t.numel() == n and t.device == lon.device
            a.d_cols[k], a.col_bytes[k] = t.data_ptr(), t.element_size()
            layout.append((name, t.dtype, t.element_size()))
            rec += t.element_size()
        a.rec_bytes = rec
        records = torch.empty((n, rec), dtype=torch.uint8, device=lon.device)
        a.d_records = records.data_ptr()
        perm = self.empty(n, torch.int32) if want_perm else None
        if perm is not None:
            a.d_perm = perm.data_ptr()
        counts = (C.c_int64 * (len(bounds) - 1))()
        a.h_counts = counts
        self._check(self.lib.od_pack_by_owner(self.ctx, C.byref(a)))
        return records, [int(c) for c in counts], layout, perm

    def unpack_records(self, records, layout):
        """records uint8 [n, rec_bytes] -> dict name -> tensor (the inverse of pack_by_owner's packing)."""
        torch = self.torch
        n = records.shape[0]
        out = {name: torch.empty(n, dtype=dt, device=records.device) for name, dt, _ in layout}
        ptrs = (C.c_void_p * len(layout))(*[out[name].data_ptr() for name, _, _ in layout])
        widths = (C.c_int32 * len(layout))(*[b for _, _, b in layout])
        self._check(self.lib.od_unpack_records(self.ctx, n, C.c_void_p(records.data_ptr()), len(layout), ptrs, widths,
                                               sum(b for _, _, b in layout)))
        return out

    def sort_by_cell(self, group, lon, lat, z=None):
        if z is not None and z.dtype != self.torch.float32:
            z = z.to(self.torch.float32)          # ordering only
        perm = self.empty(lon.numel(), self.torch.int32)
        self._check(self.lib.od_sort_by_cell(self.ctx, group.gid, lon.numel(), _ptr(lon), _ptr(lat), _ptr(z),
                                             _ptr(perm)))
        return perm

    def partition_active(self, status):
        """(perm, n_keep): stable partition of the elements by status == 0 (kept first)."""
        n = status.numel()
        perm = self.empty(n, self.torch.int32)
        nk = C.c_int64()
        self._check(self.lib.od_partition_active(self.ctx, n, _ptr(status), _ptr(perm), C.byref(nk)))
        return perm, int(nk.value)

    def permute(self, perm, src, inverse=False):
        dst = self.torch.empty_like(src)
        fn = self.lib.od_unpermute if inverse else self.lib.od_permute
        self._check(fn(self.ctx, src.numel(), _ptr(perm), _ptr(src), _ptr(dst), src.element_size()))
        return dst
