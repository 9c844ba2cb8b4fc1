"""ctypes binding of tests/emu/bspline_driver.cpp (the plan's B-spline stage compiled for the host). TEST ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_LIB = os.path.join(_HERE, "libpql_bspline_emu.so")
_lib = None


def _load():
    global _lib
    if _lib is None:
        csrc = os.path.join(_ROOT, "path_optimizer_2_b200", "csrc")
        srcs = [os.path.join(_HERE, "bspline_driver.cpp")] + [os.path.join(csrc, f) for f in (
            "pqp_plan_core.cuh", "pqp_dp_core.cuh", "pqp_bounds_core.cuh")]
        if not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _LIB, srcs[0]])
        L = C.CDLL(_LIB)
        vp, i = C.c_void_p, C.c_int
        L.bspline_emu.argtypes = [vp, vp, i, i, i, vp, vp, vp]
        L.bspline_emu_eval.argtypes = [vp, vp, i, i, vp, i, vp, vp]
        L.bspline_emu_eval.restype = None
        _lib = L
    return _lib


def _arr(v):
    return np.ascontiguousarray(v, dtype=np.float64)


def b_spline(ref_x, ref_y, cap, m_max=None):
    """-> dict(status, r, degree, x, y) as bspline_oracle.b_spline (x, y cut to r when OK, else empty)."""
    px, py = _arr(ref_x), _arr(ref_y)
    m = len(px)
    m_max = m if m_max is None else m_max
    x, y, info = np.zeros(max(cap, 1)), np.zeros(max(cap, 1)), np.zeros(2, dtype=np.int32)
    st = _load().bspline_emu(px.ctypes.data, py.ctypes.data, m, m_max, cap, x.ctypes.data, y.ctypes.data, info.ctypes.data)
    r = int(info[0]) if st == 0 else 0
    return dict(status=int(st), r=int(info[0]), degree=int(info[1]), x=x[:r].copy(), y=y[:r].copy())


def evaluate(ref_x, ref_y, degree, t):
    px, py, t = _arr(ref_x), _arr(ref_y), _arr(t)
    x, y = np.zeros(len(t)), np.zeros(len(t))
    _load().bspline_emu_eval(px.ctypes.data, py.ctypes.data, len(px), degree, t.ctypes.data, len(t), x.ctypes.data,
                             y.ctypes.data)
    return x, y
