"""TEST INFRASTRUCTURE: the host engine (tests/hostengine.py) with ShipDrift's entry point -- od_ship_step -- forwarded to the host
build of csrc/od_ship.cuh (tests/hostshim/shipdrift_shim.cpp), on top of SedimentDrift's entry points (tests/sediment_host.py).
Never imported by the product."""
import ctypes as C
import os
import subprocess
import types

import common
import sediment_host
from opendrift_b200.engine import Engine

_P = C.c_void_p
_shim = None
_HEADERS = ('od_ship.cuh', 'od_advect.cuh', 'od_interp.cuh', 'od_geod.cuh', 'od_geod_series.inc', 'od_proj.cuh')


def shim():
    """Build (once) and load tests/hostshim/libshipdrift_shim.so."""
    global _shim
    if _shim is None:
        d = os.path.join(common.ROOT, 'tests', 'hostshim')
        so, src = os.path.join(d, 'libshipdrift_shim.so'), os.path.join(d, 'shipdrift_shim.cpp')
        hdrs = [os.path.join(common.ROOT, 'opendrift_b200', 'csrc', h) for h in _HEADERS]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in [src] + hdrs):
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-shared', '-fPIC', '-o', so, src])
        lib = C.CDLL(so)
        lib.hs5_ship_step.restype = C.c_int
        lib.hs5_ship_step.argtypes = [C.c_int64, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_double, C.POINTER(C.c_int32)]
        lib.hs5_ship_wforce.restype = C.c_int
        lib.hs5_ship_wforce.argtypes = [C.c_int64, _P, _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_int32, _P, _P]
        _shim = lib
    return _shim


def install(eng):
    """Give a HostEngine ShipDrift's entry point (Engine's own wrapper over the forwarded od_* call)."""
    s, lib = shim(), eng.lib

    def od_ship_step(ctx, *args):
        lib.calls.append('od_ship_step')
        return s.hs5_ship_step(*args)

    lib.od_ship_step = od_ship_step
    eng.ship_step = types.MethodType(Engine.ship_step, eng)
    return eng


def host_engine():
    return install(sediment_host.host_engine())
