"""ctypes binding of tests/emu/collision_driver.cpp (the collision check's kernel source compiled for the host).
TEST ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

from path_optimizer_2_b200 import bounds as pb

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "libpqc_emu.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "collision_driver.cpp"),
                os.path.join(_ROOT, "path_optimizer_2_b200", "csrc", "pqp_collision_core.cuh"),
                os.path.join(_ROOT, "path_optimizer_2_b200", "csrc", "pqp_bounds_core.cuh"),
                os.path.join(_ROOT, "include", "pqp_bounds.h")]
        if not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++",
                                   "-I", os.path.join(_ROOT, "include"), "-o", _LIB, srcs[0]])
        _lib = C.CDLL(_LIB)
        _lib.pqc_emu_check.argtypes = [C.POINTER(pb.BoundsMap), C.POINTER(pb.BoundsParams), C.POINTER(pb.CollisionIn),
                                       C.POINTER(pb.CollisionOut)]
        _lib.pqc_emu_footprint.argtypes = [C.POINTER(pb.BoundsParams), C.c_void_p]
        _lib.pqc_emu_footprint.restype = None
    return _lib


def footprint(params=None):
    """-> float64 [3, 7]: x, y, r of the bounding circle and the six circles as the kernel receives them."""
    out = np.zeros((3, 7))
    lib().pqc_emu_footprint(C.byref(params if params is not None else pb.default_params()), out.ctypes.data)
    return out


def check(dist, res, poses, n, *, params=None, center=(0.0, 0.0)):
    """poses [B, rows >= 3, n_max] (contiguous) -> (first_hit [B], state_free [B, n_max], clearance [B, n_max])."""
    dist = np.ascontiguousarray(dist, dtype=np.float32)
    poses = np.ascontiguousarray(poses, dtype=np.float64)
    n = np.ascontiguousarray(n, dtype=np.int32)
    B, rows, n_max = poses.shape
    hit, free, clear = np.zeros(B, np.int32), np.zeros((B, n_max), np.uint8), np.zeros((B, n_max))
    m = pb.BoundsMap(dist.shape[0], dist.shape[1], res, center[0], center[1], dist.ctypes.data)
    p = params if params is not None else pb.default_params()
    ci = pb.CollisionIn(B, n_max, rows, poses.ctypes.data, n.ctypes.data)
    co = pb.CollisionOut(hit.ctypes.data, free.ctypes.data, clear.ctypes.data)
    assert lib().pqc_emu_check(C.byref(m), C.byref(p), C.byref(ci), C.byref(co)) == 0
    return hit, free, clear
