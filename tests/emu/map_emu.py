"""ctypes binding of tests/emu/map_driver.cpp (the distance transform's kernel source compiled for the host).
TEST ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "libpqm_emu.so")
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "map_driver.cpp"),
                os.path.join(_ROOT, "path_optimizer_2_b200", "csrc", "pqp_map_core.cuh")]
        if not os.path.exists(_LIB) or any(os.path.getmtime(s) > os.path.getmtime(_LIB) for s in srcs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++",
                                   "-o", _LIB, srcs[0]])
        _lib = C.CDLL(_LIB)
        _lib.pqm_emu_transform.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p]
    return _lib


def transform(img, res, obstacle_max=0):
    """-> (d2 int32 [rows, cols], layer float32 [rows, cols]) as the two kernels compute them."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    rows, cols = img.shape
    layer = np.zeros((rows, cols), dtype=np.float32)
    d2 = np.zeros((rows, cols), dtype=np.int32)
    rc = lib().pqm_emu_transform(img.ctypes.data, rows, cols, int(obstacle_max), float(res), layer.ctypes.data,
                                 d2.ctypes.data)
    assert rc == 0
    return d2, layer
