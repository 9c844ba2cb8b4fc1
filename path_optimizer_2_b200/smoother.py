"""ctypes binding of include/pqp_smoother.h: the reference-line smoother QPs on the GPU
(TensionSmoother2::osqpSmooth, tension_smoother_2.cpp:20-158; TensionSmoother::osqpSmooth, tension_smoother.cpp:49-177;
postSmooth's QP, reference_path_smoother.cpp:526-636), batched, one warp per QP, OSQP's algorithm in FP64. No CPU path."""
import ctypes as C

import numpy as np

from . import solver

EXPORTED_SYMBOLS = ["pqp_smoother_default_params", "pqp_smoother_create", "pqp_smoother_destroy", "pqp_tension_smooth",
                    "pqp_post_smooth", "pqp_tension_smooth_device", "pqp_post_smooth_device", "pqp_smoother_last_kernel_ms",
                    "pqp_smoother_last_error", "pqp_cartesian_tension_smooth", "pqp_cartesian_tension_smooth_device"]


class SmootherParams(C.Structure):
    _fields_ = [(n, C.c_double) for n in (
        "tension_deviation_weight", "tension_curvature_weight", "tension_curvature_rate_weight", "post_weight_x",
        "post_weight_dx", "post_weight_ddx", "rho", "sigma", "alpha", "eps_abs", "eps_rel", "eps_prim_inf", "eps_dual_inf",
        "adaptive_rho_tolerance")] + [(n, C.c_int32) for n in (
            "max_iter", "check_termination", "scaling", "adaptive_rho", "adaptive_rho_interval", "reserved")] + [
        (n, C.c_double) for n in ("cartesian_curvature_weight", "cartesian_curvature_rate_weight",
                                  "cartesian_deviation_weight")]


class TensionIn(C.Structure):
    _fields_ = [("batch", C.c_int32), ("p_max", C.c_int32)] + [(n, C.c_void_p) for n in ("p", "x", "y", "angle", "k", "s")]


class CartesianTensionIn(C.Structure):
    _fields_ = [("batch", C.c_int32), ("p_max", C.c_int32)] + [(n, C.c_void_p) for n in ("p", "x", "y", "angle", "clearance")]


class TensionOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("x", "y", "s", "status", "iters", "x_full")]


class PostIn(C.Structure):
    _fields_ = [("batch", C.c_int32), ("p_max", C.c_int32)] + [(n, C.c_void_p) for n in ("p", "layer_s", "lower", "upper", "vehicle_l")]


class PostOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("offsets", "status", "iters", "x_full")]


def _lib():
    L = solver.load_library()
    if not getattr(L, "_smoother_declared", False):
        vp = C.c_void_p
        L.pqp_smoother_default_params.argtypes = [C.POINTER(SmootherParams)]
        L.pqp_smoother_default_params.restype = None
        L.pqp_smoother_create.argtypes = [C.POINTER(SmootherParams), C.c_int32, C.c_int32, C.c_int32, C.POINTER(vp)]
        L.pqp_smoother_destroy.argtypes = [vp]
        L.pqp_smoother_destroy.restype = None
        L.pqp_tension_smooth.argtypes = [vp, C.POINTER(TensionIn), C.POINTER(TensionOut)]
        L.pqp_post_smooth.argtypes = [vp, C.POINTER(PostIn), C.POINTER(PostOut)]
        L.pqp_tension_smooth_device.argtypes = [vp, C.POINTER(TensionIn), C.POINTER(TensionOut), vp]
        L.pqp_post_smooth_device.argtypes = [vp, C.POINTER(PostIn), C.POINTER(PostOut), vp]
        L.pqp_cartesian_tension_smooth.argtypes = [vp, C.POINTER(CartesianTensionIn), C.POINTER(TensionOut)]
        L.pqp_cartesian_tension_smooth_device.argtypes = [vp, C.POINTER(CartesianTensionIn), C.POINTER(TensionOut), vp]
        L.pqp_smoother_last_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
        L.pqp_smoother_last_error.argtypes = [vp]
        L.pqp_smoother_last_error.restype = C.c_char_p
        L._smoother_declared = True
    return L


def default_params():
    p = SmootherParams()
    _lib().pqp_smoother_default_params(C.byref(p))
    return p


def _pad(rows, p_max):
    out = np.zeros((len(rows), p_max))
    for b, r in enumerate(rows):
        out[b, :len(r)] = r
    return out


class Smoother:
    def __init__(self, *, p_max, batch_max, device=0, params=None):
        self.L = _lib()
        self.params = params or default_params()
        self.p_max, self.batch_max = int(p_max), int(batch_max)
        h = C.c_void_p()
        rc = self.L.pqp_smoother_create(C.byref(self.params), self.p_max, self.batch_max, int(device), C.byref(h))
        if rc:
            raise solver.PqpError(rc, (self.L.pqp_smoother_last_error(None) or b"").decode())
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.pqp_smoother_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc:
            raise solver.PqpError(rc, (self.L.pqp_smoother_last_error(self.h) or b"").decode())

    def tension(self, xs, ys, angles, ks, ss, full=False):
        """Lists of per-path arrays -> dict of padded result arrays (TensionSmoother2::osqpSmooth)."""
        B = len(xs)
        p = np.array([len(v) for v in xs], dtype=np.int32)
        arr = [_pad(v, self.p_max) for v in (xs, ys, angles, ks, ss)]
        rx, ry, rs = (np.zeros((B, self.p_max)) for _ in range(3))
        status, iters = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        xf = np.zeros((B, 4 * self.p_max)) if full else None
        tin = TensionIn(B, self.p_max, p.ctypes.data, *(a.ctypes.data for a in arr))
        tout = TensionOut(rx.ctypes.data, ry.ctypes.data, rs.ctypes.data, status.ctypes.data, iters.ctypes.data,
                          None if xf is None else xf.ctypes.data)
        self._check(self.L.pqp_tension_smooth(self.h, C.byref(tin), C.byref(tout)))
        return dict(p=p, x=rx, y=ry, s=rs, status=status, iters=iters, x_full=xf)

    def cartesian_tension(self, xs, ys, angles, clearances, full=False):
        """Lists of per-path arrays -> dict of padded result arrays (TensionSmoother::osqpSmooth). `clearances`: the
        map's obstacle distance at each point (Map::getObstacleDistance, 0 off the map). x_full [B][3 p_max]: x block,
        y block, d block."""
        B = len(xs)
        p = np.array([len(v) for v in xs], dtype=np.int32)
        arr = [_pad(v, self.p_max) for v in (xs, ys, angles, clearances)]
        rx, ry, rs = (np.zeros((B, self.p_max)) for _ in range(3))
        status, iters = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        xf = np.zeros((B, 3 * self.p_max)) if full else None
        cin = CartesianTensionIn(B, self.p_max, p.ctypes.data, *(a.ctypes.data for a in arr))
        cout = TensionOut(rx.ctypes.data, ry.ctypes.data, rs.ctypes.data, status.ctypes.data, iters.ctypes.data,
                          None if xf is None else xf.ctypes.data)
        self._check(self.L.pqp_cartesian_tension_smooth(self.h, C.byref(cin), C.byref(cout)))
        return dict(p=p, x=rx, y=ry, s=rs, status=status, iters=iters, x_full=xf)

    def cartesian_tension_device(self, p, x, y, angle, clearance, *, full=False, stream=None):
        """Device call on torch tensors (cuda, contiguous): p int32 [B], x / y / angle / clearance float64 [B][p_max].
        Asynchronous on `stream` (default: the current stream); returns a dict of output tensors."""
        import torch
        B, dev = int(p.shape[0]), p.device
        for t in (p, x, y, angle, clearance):
            assert t.is_cuda and t.is_contiguous()
        z = lambda *shape: torch.zeros(shape, dtype=torch.float64, device=dev)  # noqa: E731
        out = dict(x=z(B, self.p_max), y=z(B, self.p_max), s=z(B, self.p_max),
                   status=torch.zeros(B, dtype=torch.int32, device=dev), iters=torch.zeros(B, dtype=torch.int32, device=dev),
                   x_full=z(B, 3 * self.p_max) if full else None)
        cin = CartesianTensionIn(B, self.p_max, *(t.data_ptr() for t in (p, x, y, angle, clearance)))
        cout = TensionOut(*(out[k].data_ptr() for k in ("x", "y", "s", "status", "iters")),
                          None if out["x_full"] is None else out["x_full"].data_ptr())
        s = stream if stream is not None else torch.cuda.current_stream(dev)
        self._check(self.L.pqp_cartesian_tension_smooth_device(self.h, C.byref(cin), C.byref(cout), C.c_void_p(s.cuda_stream)))
        return out

    def post(self, layer_s, lower, upper, vehicle_l, full=False):
        """postSmooth's QP for lists of per-path layer arrays -> lateral offsets per layer."""
        B = len(layer_s)
        p = np.array([len(v) for v in layer_s], dtype=np.int32)
        arr = [_pad(v, self.p_max) for v in (layer_s, lower, upper)]
        vl = np.ascontiguousarray(vehicle_l, dtype=np.float64)
        off = np.zeros((B, self.p_max))
        status, iters = np.zeros(B, dtype=np.int32), np.zeros(B, dtype=np.int32)
        xf = np.zeros((B, 3 * self.p_max)) if full else None
        pin = PostIn(B, self.p_max, p.ctypes.data, *(a.ctypes.data for a in arr), vl.ctypes.data)
        pout = PostOut(off.ctypes.data, status.ctypes.data, iters.ctypes.data, None if xf is None else xf.ctypes.data)
        self._check(self.L.pqp_post_smooth(self.h, C.byref(pin), C.byref(pout)))
        return dict(p=p, offsets=off, status=status, iters=iters, x_full=xf)

    @property
    def last_kernel_ms(self):
        ms = C.c_float()
        self._check(self.L.pqp_smoother_last_kernel_ms(self.h, C.byref(ms)))
        return ms.value
