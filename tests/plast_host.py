"""TEST INFRASTRUCTURE: the host engine (tests/hostengine.py) with PlastDrift's entry point -- od_plast_step -- forwarded to the host
build of csrc/od_plast.cuh (tests/hostshim/plast_shim.cpp), on top of SedimentDrift's entry points (tests/sediment_host.py), which
bring the mixing launch and the tabularised Stokes drift.  Never imported by the product."""
import ctypes as C
import glob
import os
import subprocess
import types

import common
import sediment_host
from opendrift_b200.engine import Engine

_P = C.c_void_p
_shim = None


def shim():
    """Build (once) and load tests/hostshim/libplast_shim.so."""
    global _shim
    if _shim is None:
        d = os.path.join(common.ROOT, 'tests', 'hostshim')
        so, src = os.path.join(d, 'libplast_shim.so'), os.path.join(d, 'plast_shim.cpp')
        deps = [src] + glob.glob(os.path.join(common.ROOT, 'opendrift_b200', 'csrc', '*.cuh')) + \
            glob.glob(os.path.join(common.ROOT, 'opendrift_b200', 'csrc', '*.inc'))
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in deps):
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-shared', '-fPIC', '-o', so, src])
        lib = C.CDLL(so)
        lib.hs6_plast_step.restype = C.c_int
        lib.hs6_plast_step.argtypes = [C.c_int64, _P, _P, _P, _P, C.c_int32, _P, _P, _P, C.c_int32, _P, _P, C.c_uint64, C.c_int32, _P, C.c_int32,
                                       C.c_int32, _P, _P, _P, C.c_int32, C.c_double, C.c_double, C.POINTER(C.c_int32)]
        lib.hs6_philox_u0.restype = C.c_int
        lib.hs6_philox_u0.argtypes = [C.c_int64, C.c_uint64, _P, C.c_int32, C.c_uint32, _P]
        _shim = lib
    return _shim


def install(eng):
    """Give a HostEngine PlastDrift's entry point (Engine's own wrapper over the forwarded od_* call)."""
    s, lib = shim(), eng.lib

    def od_plast_step(ctx, *args):
        lib.calls.append('od_plast_step')
        return s.hs6_plast_step(*args)

    lib.od_plast_step = od_plast_step
    eng.plast_step = types.MethodType(Engine.plast_step, eng)
    return eng


def host_engine():
    return install(sediment_host.host_engine())
