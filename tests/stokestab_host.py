"""TEST INFRASTRUCTURE: the host engine (tests/hostengine.py) with the entry point of drift:use_tabularised_stokes_drift --
od_stokes_parameterised -- forwarded to the host build of csrc/od_stokes.cuh (tests/hostshim/stokestab_shim.cpp), on top of the
sea-level entry points (tests/sealevel_host.py).  Never imported by the product."""
import ctypes as C
import os
import subprocess
import types

import common
import sealevel_host
from opendrift_b200.engine import Engine

_P = C.c_void_p
_shim = None
_HEADERS = ('od_stokes.cuh', 'od_advect.cuh', 'od_interp.cuh', 'od_geod.cuh', 'od_geod_series.inc', 'od_proj.cuh')


def shim():
    """Build (once) and load tests/hostshim/libstokestab_shim.so."""
    global _shim
    if _shim is None:
        d = os.path.join(common.ROOT, 'tests', 'hostshim')
        so, src = os.path.join(d, 'libstokestab_shim.so'), os.path.join(d, 'stokestab_shim.cpp')
        hdrs = [os.path.join(common.ROOT, 'opendrift_b200', 'csrc', h) for h in _HEADERS]
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in [src] + hdrs):
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-shared', '-fPIC', '-o', so, src])
        lib = C.CDLL(so)
        lib.hs3_stokes_parameterised.restype = C.c_int
        lib.hs3_stokes_parameterised.argtypes = [C.c_int64, _P, _P, _P, C.c_int32, _P, C.c_int32, _P, _P, _P]
        _shim = lib
    return _shim


def install(eng):
    """Give a HostEngine the tabularised Stokes drift entry point (Engine's own wrapper over the forwarded od_* call)."""
    s, lib = shim(), eng.lib

    def od_stokes_parameterised(ctx, *args):
        lib.calls.append('od_stokes_parameterised')
        return s.hs3_stokes_parameterised(*args)

    lib.od_stokes_parameterised = od_stokes_parameterised
    eng.stokes_parameterised = types.MethodType(Engine.stokes_parameterised, eng)
    return eng


def host_engine():
    return install(sealevel_host.host_engine())
