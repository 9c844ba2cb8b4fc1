"""ctypes binding of tests/emu/boxes_driver.cpp (the obstacle-box stamping and the distance transform's kernel source
compiled for the host). TEST ONLY."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_SRCS = [os.path.join(_HERE, "boxes_driver.cpp"), os.path.join(_ROOT, "path_optimizer_2_b200", "csrc", "pqp_map_core.cuh")]
_lib = None


def lib():
    """Compiled into a temporary directory on first use, so a read-only tree works too."""
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="pqm_boxes_emu_"), "libpqm_boxes_emu.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-x", "c++",
                               "-o", out, _SRCS[0]])
        _lib = C.CDLL(out)
        vp = C.c_void_p
        _lib.pqm_emu_boxes_transform.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double,
                                                 vp, C.c_int, vp, vp]
        _lib.pqm_emu_boxes_mask.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, vp, C.c_int, vp]
    return _lib


def _boxes(boxes):
    return np.ascontiguousarray(np.asarray(boxes, dtype=np.float64).reshape(-1, 5))


def transform(img, res, center, boxes, obstacle_max=0):
    """-> (d2 int32 [rows, cols], layer float32 [rows, cols]) of the base image plus boxes [k, 5], as the kernels
    compute them."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    bx = _boxes(boxes)
    rows, cols = img.shape
    layer = np.zeros((rows, cols), dtype=np.float32)
    d2 = np.zeros((rows, cols), dtype=np.int32)
    rc = lib().pqm_emu_boxes_transform(img.ctypes.data, rows, cols, int(obstacle_max), float(res), float(center[0]),
                                       float(center[1]), bx.ctypes.data, len(bx), layer.ctypes.data, d2.ctypes.data)
    assert rc == 0
    return d2, layer


def mask(shape, res, center, boxes):
    """bool [rows, cols]: the predicate over every cell, no base image."""
    bx = _boxes(boxes)
    out = np.zeros(shape, dtype=np.uint8)
    lib().pqm_emu_boxes_mask(shape[0], shape[1], float(res), float(center[0]), float(center[1]), bx.ctypes.data,
                             len(bx), out.ctypes.data)
    return out.astype(bool)
