"""ctypes binding of include/pqp_dp.h: the lattice DP search of the reference's front end
(ReferencePathSmoother::graphSearchDp, reference_path_smoother.cpp:142-295) for a batch of paths over
the shared obstacle map held by a `bounds.PathBounds` handle. No CPU path."""
import ctypes as C

import numpy as np

from . import solver

EXPORTED_SYMBOLS = ["pqp_dp_default_params", "pqp_dp_create", "pqp_dp_destroy", "pqp_dp_lateral_count", "pqp_dp_search",
                    "pqp_dp_search_device", "pqp_dp_last_kernel_ms", "pqp_dp_last_error", "pqp_dp_search_mapped",
                    "pqp_dp_search_mapped_device"]
DP_OK, DP_VEHICLE_FAR, DP_TOO_MANY_LAYERS, DP_MAP_INDEX = 1, 0, -1, -2


class DpParams(C.Structure):
    _fields_ = [("lateral_range", C.c_double), ("lateral_spacing", C.c_double), ("longitudinal_spacing", C.c_double),
                ("car_width", C.c_double)]


class DpIn(C.Structure):
    _fields_ = [("batch", C.c_int32), ("k_max", C.c_int32), ("spline", C.c_void_p), ("k", C.c_void_p),
                ("length", C.c_void_p), ("start", C.c_void_p)]


class DpOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("status", "n_layers", "n_out", "layer_s", "lower", "upper", "chosen", "vehicle_l",
                                          "target_s", "cost", "parent", "feasible")]


def _lib():
    L = solver.load_library()
    if not getattr(L, "_dp_declared", False):
        vp = C.c_void_p
        L.pqp_dp_default_params.argtypes = [C.POINTER(DpParams)]
        L.pqp_dp_default_params.restype = None
        L.pqp_dp_create.argtypes = [vp, C.POINTER(DpParams), C.c_int32, C.c_int32, C.POINTER(vp)]
        L.pqp_dp_destroy.argtypes = [vp]
        L.pqp_dp_destroy.restype = None
        L.pqp_dp_lateral_count.argtypes = [vp]
        L.pqp_dp_lateral_count.restype = C.c_int32
        L.pqp_dp_search.argtypes = [vp, C.POINTER(DpIn), C.POINTER(DpOut)]
        L.pqp_dp_search_device.argtypes = [vp, C.POINTER(DpIn), C.POINTER(DpOut), vp]
        L.pqp_dp_search_mapped.argtypes = [vp, C.POINTER(DpIn), vp, C.POINTER(DpOut)]
        L.pqp_dp_search_mapped_device.argtypes = [vp, C.POINTER(DpIn), vp, C.POINTER(DpOut), vp]
        L.pqp_dp_last_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
        L.pqp_dp_last_error.argtypes = [vp]
        L.pqp_dp_last_error.restype = C.c_char_p
        L._dp_declared = True
    return L


def default_params():
    p = DpParams()
    p.lateral_range, p.lateral_spacing, p.longitudinal_spacing, p.car_width = 10.0, 0.6, 1.5, 2.0
    return p


class DpResult:
    def __init__(self, batch, layers_max, lateral, tables=True):
        self.status, self.n_layers, self.n_out = (np.zeros(batch, dtype=np.int32) for _ in range(3))
        self.layer_s, self.lower, self.upper = (np.zeros((batch, layers_max)) for _ in range(3))
        self.chosen = np.zeros((batch, layers_max), dtype=np.int32)
        self.vehicle_l, self.target_s = np.zeros(batch), np.zeros(batch)
        self.cost = np.zeros((batch, layers_max, lateral)) if tables else None
        self.parent = np.zeros((batch, layers_max, lateral), dtype=np.int8) if tables else None
        self.feasible = np.zeros((batch, layers_max, lateral), dtype=np.uint8) if tables else None

    def as_struct(self):
        p = lambda a: None if a is None else a.ctypes.data  # noqa: E731
        return DpOut(p(self.status), p(self.n_layers), p(self.n_out), p(self.layer_s), p(self.lower), p(self.upper),
                     p(self.chosen), p(self.vehicle_l), p(self.target_s), p(self.cost), p(self.parent), p(self.feasible))


class DpSearch:
    """graphSearchDp for a batch; `path_bounds` (bounds.PathBounds) owns the map and must outlive this."""

    def __init__(self, path_bounds, *, layers_max=160, batch_max, params=None):
        self.L = _lib()
        self.owner = path_bounds
        self.params = params or default_params()
        self.layers_max, self.batch_max = int(layers_max), int(batch_max)
        h = C.c_void_p()
        rc = self.L.pqp_dp_create(path_bounds.h, C.byref(self.params), self.layers_max, self.batch_max, C.byref(h))
        if rc:
            raise solver.PqpError(rc, (self.L.pqp_dp_last_error(None) or b"").decode())
        self.h = h
        self.lateral = self.L.pqp_dp_lateral_count(h)

    def close(self):
        if getattr(self, "h", None):
            self.L.pqp_dp_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc:
            raise solver.PqpError(rc, (self.L.pqp_dp_last_error(self.h) or b"").decode())

    def search(self, spline, k, length, start, tables=True, map_index=None) -> DpResult:
        """`map_index` [b]: path b on map slot map_index[b] of the owner (out of range: status DP_MAP_INDEX)."""
        spline = np.ascontiguousarray(spline, dtype=np.float64)
        k = np.ascontiguousarray(k, dtype=np.int32)
        length = np.ascontiguousarray(length, dtype=np.float64)
        start = np.ascontiguousarray(start, dtype=np.float64)
        B, k_max = spline.shape[0], spline.shape[2]
        res = DpResult(B, self.layers_max, self.lateral, tables)
        din = DpIn(B, k_max, spline.ctypes.data, k.ctypes.data, length.ctypes.data, start.ctypes.data)
        dout = res.as_struct()
        if map_index is None:
            self._check(self.L.pqp_dp_search(self.h, C.byref(din), C.byref(dout)))
        else:
            idx = np.ascontiguousarray(map_index, dtype=np.int32)
            assert idx.shape == (B,)
            self._check(self.L.pqp_dp_search_mapped(self.h, C.byref(din), idx.ctypes.data, C.byref(dout)))
        return res

    def search_device(self, din: DpIn, dout: DpOut, stream=0):
        self._check(self.L.pqp_dp_search_device(self.h, C.byref(din), C.byref(dout), C.c_void_p(stream)))

    @property
    def last_kernel_ms(self):
        ms = C.c_float()
        self._check(self.L.pqp_dp_last_kernel_ms(self.h, C.byref(ms)))
        return ms.value
