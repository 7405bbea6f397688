"""TEST INFRASTRUCTURE: the host engine (tests/hostengine.py) with LarvalFish's entry points -- od_larval_develop and
od_larval_migrate -- forwarded to the host build of csrc/od_larval.cuh (tests/hostshim/larval_shim.cpp), on top of SedimentDrift's
entry points (tests/sediment_host.py), which bring the mixing launch and the tabularised Stokes drift.  Never imported by the
product."""
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
    """Build (once) and load tests/hostshim/liblarval_shim.so."""
    global _shim
    if _shim is None:
        d = os.path.join(common.ROOT, 'tests', 'hostshim')
        so, src = os.path.join(d, 'liblarval_shim.so'), os.path.join(d, 'larval_shim.cpp')
        deps = [src] + glob.glob(os.path.join(common.ROOT, 'opendrift_b200', 'csrc', '*.cuh'))
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in deps):
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-shared', '-fPIC', '-o', so, src])
        lib = C.CDLL(so)
        lib.hs7_larval_develop.restype = C.c_int
        lib.hs7_larval_develop.argtypes = [C.c_int64, _P, _P, _P, C.c_int32, _P, C.c_int32, _P, C.c_int32, _P, C.c_int32, _P, C.c_int32, _P,
                                           C.c_int32, C.c_int32, _P, C.c_double, C.POINTER(C.c_int32)]
        lib.hs7_larval_migrate.restype = C.c_int
        lib.hs7_larval_migrate.argtypes = [C.c_int64, _P, C.c_int32, _P, C.c_int32, _P, C.c_int32, C.c_double, C.c_double, C.c_double]
        _shim = lib
    return _shim


def install(eng):
    """Give a HostEngine LarvalFish's entry points (Engine's own wrappers over the forwarded od_* calls)."""
    s, lib = shim(), eng.lib

    def od_larval_develop(ctx, *args):
        lib.calls.append('od_larval_develop')
        return s.hs7_larval_develop(*args)

    def od_larval_migrate(ctx, *args):
        lib.calls.append('od_larval_migrate')
        return s.hs7_larval_migrate(*args)

    lib.od_larval_develop = od_larval_develop
    lib.od_larval_migrate = od_larval_migrate
    for name in ('larval_develop', 'larval_migrate'):
        setattr(eng, name, types.MethodType(getattr(Engine, name), eng))
    for name in ('LARVAL_STAGED', 'LARVAL_HOT', 'LARVAL_NAN_T'):
        setattr(eng, name, getattr(Engine, name))
    return eng


def host_engine():
    return install(sediment_host.host_engine())
