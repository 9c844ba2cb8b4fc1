"""ctypes binding of tests/emu/plan_driver.cpp (the plan glue's per-path source compiled for the host). TEST ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_LIB = os.path.join(_HERE, "libpql_emu.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        csrc = os.path.join(_ROOT, "path_optimizer_2_b200", "csrc")
        srcs = [os.path.join(_HERE, "plan_driver.cpp")] + [os.path.join(csrc, f) for f in (
            "pqp_plan_core.cuh", "pqp_dp_core.cuh", "pqp_bounds_core.cuh")]
        if not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _LIB, srcs[0]])
        L = C.CDLL(_LIB)
        vp, d, i = C.c_void_p, C.c_double, C.c_int
        L.plan_emu_fit.argtypes = [vp, vp, i, vp, vp, vp]
        L.plan_emu_fit.restype = None
        L.plan_emu_chord.argtypes = [vp, vp, i, vp]
        L.plan_emu_segment_count.argtypes = [d, i]
        L.plan_emu_segment.argtypes = [vp, i, i, i, vp]
        L.plan_emu_segment.restype = None
        L.plan_emu_post_points.argtypes = [vp, i, i, vp, vp, i, vp, vp, vp]
        L.plan_emu_post_points.restype = None
        L.plan_emu_process.argtypes = [vp, i, i, d, vp, vp, d, vp]
        L.plan_emu_precise.argtypes = [vp, i, i, d]
        L.plan_emu_end_heading.argtypes = [i, i, d, d, vp]
        L.plan_emu_end_heading.restype = None
        L.plan_emu_placeholder.argtypes = [vp, vp, vp]
        L.plan_emu_placeholder.restype = None
        _lib = L
    return _lib


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def fit(sx, y):
    """-> (a, b, c) of one coordinate."""
    sx, y = _f64(sx), _f64(y)
    a, b, c = np.zeros(len(sx)), np.zeros(len(sx)), np.zeros(len(sx))
    lib().plan_emu_fit(sx.ctypes.data, y.ctypes.data, len(sx), a.ctypes.data, b.ctypes.data, c.ctypes.data)
    return a, b, c


def spline_rows(s, x, y):
    """[9][k] rows as the kernels fit them."""
    rows = [_f64(s)]
    for v in (x, y):
        rows += list(fit(s, v)) + [_f64(v)]
    return np.ascontiguousarray(np.stack(rows))


def chord(x, y):
    x, y = _f64(x), _f64(y)
    s = np.zeros(len(x))
    ok = lib().plan_emu_chord(x.ctypes.data, y.ctypes.data, len(x), s.ctypes.data)
    return s, bool(ok)


def segment_count(max_s, cap=1 << 20):
    return lib().plan_emu_segment_count(float(max_s), int(cap))


def segment(rows, p):
    """-> (x, y, angle, k, s) of samples 0 .. p-1."""
    rows = _f64(rows)
    out = np.zeros((5, p))
    lib().plan_emu_segment(rows.ctypes.data, rows.shape[1], rows.shape[1], p, out.ctypes.data)
    return tuple(out)


def post_points(rows, layer_s, offsets):
    rows, layer_s, offsets = _f64(rows), _f64(layer_s), _f64(offsets)
    n = len(layer_s)
    s, x, y = np.zeros(n), np.zeros(n), np.zeros(n)
    lib().plan_emu_post_points(rows.ctypes.data, rows.shape[1], rows.shape[1], layer_s.ctypes.data, offsets.ctypes.data,
                               n, s.ctypes.data, x.ctypes.data, y.ctypes.data)
    return s, x, y


def process(rows, length, start, target, epsilon=1e-6):
    """-> (status, l0, psi0, max_s)."""
    rows, start, target = _f64(rows), _f64(start), _f64(target)
    out = np.zeros(3)
    st = lib().plan_emu_process(rows.ctypes.data, rows.shape[1], rows.shape[1], float(length), start.ctypes.data,
                                target.ctypes.data, float(epsilon), out.ctypes.data)
    return st, out[0], out[1], out[2]


def precise(s, rough, precise_length=30.0):
    s = _f64(s)
    return lib().plan_emu_precise(s.ctypes.data, len(s), 1 if rough else 0, float(precise_length))


def end_heading(constrain, blocked, target_heading, last_heading):
    out = np.zeros(2)
    lib().plan_emu_end_heading(1 if constrain else 0, 1 if blocked else 0, float(target_heading), float(last_heading),
                               out.ctypes.data)
    return out[0], out[1]


def placeholder():
    s, x, y = np.zeros(3), np.zeros(3), np.zeros(3)
    lib().plan_emu_placeholder(s.ctypes.data, x.ctypes.data, y.ctypes.data)
    return s, x, y
