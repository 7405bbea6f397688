"""TEST INFRASTRUCTURE: the host engine (tests/hostengine.py) with the sea-level entry points of the library -- od_store_previous_env
and od_vertical_advection_corrected -- forwarded to the host build of csrc/od_sealevel.cuh (tests/hostshim/sealevel_shim.cpp).
Never imported by the product."""
import ctypes as C
import glob
import os
import subprocess
import types

import common
from hostengine import HostEngine
from opendrift_b200.engine import Engine

_P = C.c_void_p
_shim = None


def shim():
    """Build (once) and load tests/hostshim/libsealevel_shim.so."""
    global _shim
    if _shim is None:
        d = os.path.join(common.ROOT, 'tests', 'hostshim')
        so, src = os.path.join(d, 'libsealevel_shim.so'), os.path.join(d, 'sealevel_shim.cpp')
        hdrs = glob.glob(os.path.join(common.ROOT, 'opendrift_b200', 'csrc', 'od_sealevel.cuh'))
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in [src] + hdrs):
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-shared', '-fPIC', '-o', so, src])
        lib = C.CDLL(so)
        lib.hs2_store_previous_env.restype = C.c_int
        lib.hs2_store_previous_env.argtypes = [C.c_int64, _P, _P, _P, C.c_int32, C.c_double, C.c_int32, C.c_int64, _P, _P]
        lib.hs2_vertical_advection_corrected.restype = C.c_int
        lib.hs2_vertical_advection_corrected.argtypes = [C.c_int64, _P, C.c_int32, _P, _P, _P, _P, C.c_float, _P, C.c_int32,
                                                         C.c_double]
        _shim = lib
    return _shim


def install(eng):
    """Give a HostEngine the sea-level entry points (Engine's own wrappers over the forwarded od_* calls)."""
    s, lib = shim(), eng.lib

    def od_store_previous_env(ctx, *args):
        lib.calls.append('od_store_previous_env')
        return s.hs2_store_previous_env(*args)

    def od_vertical_advection_corrected(ctx, *args):
        lib.calls.append('od_vertical_advection_corrected')
        return s.hs2_vertical_advection_corrected(*args)

    lib.od_store_previous_env = od_store_previous_env
    lib.od_vertical_advection_corrected = od_vertical_advection_corrected
    eng.store_previous_env = types.MethodType(Engine.store_previous_env, eng)
    eng.vertical_advection_corrected = types.MethodType(Engine.vertical_advection_corrected, eng)
    return eng


def host_engine():
    return install(HostEngine())
