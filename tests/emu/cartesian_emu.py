"""ctypes binding of tests/emu/cartesian_driver.cpp (the Cartesian tension QP of the CUDA library on the CPU). TEST ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

from .smoother_emu import DEFAULT_SETTINGS

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_LIB = os.path.join(_HERE, "libpqs_cartesian_emu.so")
_lib = None


def _load():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "cartesian_driver.cpp"),
                os.path.join(_ROOT, "path_optimizer_2_b200", "csrc", "pqp_smoother_core.cuh")]
        if not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _LIB, srcs[0]])
        _lib = C.CDLL(_LIB)
        _lib.cartesian_emu.argtypes = [C.c_int] + [C.c_void_p] * 11
    return _lib


def _arr(v):
    return np.ascontiguousarray(v, dtype=np.float64)


def cartesian(x, y, a, clearance, weights=(1.0, 50.0, 0.0), settings=DEFAULT_SETTINGS):
    """TensionSmoother::osqpSmooth; weights: curvature, curvature rate, deviation."""
    L = _load()
    x, y, a, cl = (_arr(v) for v in (x, y, a, clearance))
    p = len(x)
    rx, ry, rs, xf, info = np.zeros(p), np.zeros(p), np.zeros(p), np.zeros(3 * p), np.zeros(6)
    w, st = _arr(weights), _arr(settings)
    L.cartesian_emu(p, *(v.ctypes.data for v in (x, y, a, cl, w, st, rx, ry, rs, xf, info)))
    return dict(status=int(info[0]), iters=int(info[1]), rho_updates=int(info[2]), pri_res=info[3], dua_res=info[4], obj=info[5],
                x=rx, y=ry, s=rs, x_full=xf)
