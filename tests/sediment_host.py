"""TEST INFRASTRUCTURE: the host engine (tests/hostengine.py) with SedimentDrift's entry points -- od_vertical_mixing_settle and
od_resuspend -- forwarded to the host build of csrc/od_mix.cuh (tests/hostshim/sediment_shim.cpp), on top of the sea-level and
tabularised Stokes entry points (tests/stokestab_host.py).  Never imported by the product."""
import ctypes as C
import glob
import os
import subprocess
import types

import common
import stokestab_host
from opendrift_b200 import _lib
from opendrift_b200.engine import Engine

_P = C.c_void_p
_shim = None


def shim():
    """Build (once) and load tests/hostshim/libsediment_shim.so."""
    global _shim
    if _shim is None:
        d = os.path.join(common.ROOT, 'tests', 'hostshim')
        so, src = os.path.join(d, 'libsediment_shim.so'), os.path.join(d, 'sediment_shim.cpp')
        deps = [src, os.path.join(d, 'hostshim.cpp')] + glob.glob(os.path.join(common.ROOT, 'opendrift_b200', 'csrc', '*.cuh')) + \
            glob.glob(os.path.join(common.ROOT, 'opendrift_b200', 'csrc', '*.inc'))
        if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(f) for f in deps):
            subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-shared', '-fPIC', '-o', so, src], cwd=d)
        lib = C.CDLL(so)
        HG, HP = C.POINTER(common.HsGroup), C.POINTER(common.HsPair)
        lib.hs4_mix_settle.restype = C.c_int
        lib.hs4_mix_settle.argtypes = [C.POINTER(_lib.MixArgs), HG, HP, _P, _P, C.POINTER(C.c_int64)]
        lib.hs4_resuspend.restype = C.c_int
        lib.hs4_resuspend.argtypes = [C.c_int64, _P, _P, C.c_float, _P, _P, C.c_int32]
        _shim = lib
    return _shim


def install(eng):
    """Give a HostEngine SedimentDrift's entry points (Engine's own wrappers over the forwarded od_* calls)."""
    s, lib = shim(), eng.lib

    def od_vertical_mixing_settle(ctx, args, moving_out, status_out, h_undecided):
        lib.calls.append('od_vertical_mixing_settle')
        a = args._obj
        if a.model == _lib.OD_MIX_ENVIRONMENT:
            g, pr = lib._gp(a.group_k, a.t_k)
            return s.hs4_mix_settle(args, g, C.byref(pr), moving_out, status_out, h_undecided)
        return s.hs4_mix_settle(args, None, None, moving_out, status_out, h_undecided)

    def od_resuspend(ctx, *args):
        lib.calls.append('od_resuspend')
        return s.hs4_resuspend(*args)

    lib.od_vertical_mixing_settle = od_vertical_mixing_settle
    lib.od_resuspend = od_resuspend
    eng.vertical_mixing_settle = types.MethodType(Engine.vertical_mixing_settle, eng)
    eng.resuspend = types.MethodType(Engine.resuspend, eng)
    return eng


def host_engine():
    return install(stokestab_host.host_engine())

