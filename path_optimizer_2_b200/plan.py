"""ctypes binding of include/pqp_plan.h: PathOptimizer::solve (path_optimizer.cpp:34-71) for a batch of paths on the
GPU, from the bSpline() samples of each path to its final path. `Planner` owns one handle: the map, the stage handles
and all scratch. No CPU path."""
import ctypes as C

import numpy as np

from . import abi, bounds, dp, smoother, solver

EXPORTED_SYMBOLS = ["pqp_plan_default_params", "pqp_plan_create", "pqp_plan_destroy", "pqp_plan", "pqp_plan_device",
                    "pqp_plan_last_stage_ms", "pqp_plan_launch_count", "pqp_plan_last_error"]

STATUS_NAMES = ("OK", "SPLINE_DEGENERATE", "TOO_MANY_POINTS", "TENSION_FAILED", "DP_VEHICLE_FAR", "POST_TOO_SHORT",
                "POST_FAILED", "EMPTY_REFERENCE", "INIT_HEADING", "TOO_MANY_KNOTS", "BLOCKED_AT_START",
                "PRE_SOLVE_FAILED", "SOLVE_FAILED")
(OK, SPLINE_DEGENERATE, TOO_MANY_POINTS, TENSION_FAILED, DP_VEHICLE_FAR, POST_TOO_SHORT, POST_FAILED, EMPTY_REFERENCE,
 INIT_HEADING, TOO_MANY_KNOTS, BLOCKED_AT_START, PRE_SOLVE_FAILED, SOLVE_FAILED) = range(13)
PATH_ROWS = ("x", "y", "heading", "k", "d_k", "l", "d_heading")
STAGES = ("smoothing", "segmentation", "optimisation", "total")
# PlanParams.smoothing_method: the reference's --smoothing_method
SMOOTH_TENSION2, SMOOTH_TENSION = 0, 1
SMOOTHING_METHODS = {"TENSION2": SMOOTH_TENSION2, "TENSION": SMOOTH_TENSION}


class PlanParams(C.Structure):
    _fields_ = [("solver", abi.PqpParams), ("bounds", bounds.BoundsParams), ("dp", dp.DpParams),
                ("smoother", smoother.SmootherParams), ("output_spacing", C.c_double),
                ("precise_planning_length", C.c_double), ("dynamic_segmentation", C.c_int32),
                ("rough_constraints_far_away", C.c_int32), ("constraint_end_heading", C.c_int32),
                ("smoothing_method", C.c_int32)]


class PlanIn(C.Structure):
    _fields_ = [("batch", C.c_int32), ("r_max", C.c_int32)] + [
        (n, C.c_void_p) for n in ("raw_x", "raw_y", "r", "start", "target")]


# (name, dtype, shape given (P, L, N, R)) in the order of pqp_plan_trace
_TRACE = [
    ("raw_spline", np.float64, lambda P, L, N, R: (9, R)), ("seg_p", np.int32, lambda *d: ()),
    ("seg_x", np.float64, lambda P, L, N, R: (P,)), ("seg_y", np.float64, lambda P, L, N, R: (P,)),
    ("seg_angle", np.float64, lambda P, L, N, R: (P,)), ("seg_k", np.float64, lambda P, L, N, R: (P,)),
    ("seg_s", np.float64, lambda P, L, N, R: (P,)),
    ("tension_x", np.float64, lambda P, L, N, R: (P,)), ("tension_y", np.float64, lambda P, L, N, R: (P,)),
    ("tension_s", np.float64, lambda P, L, N, R: (P,)), ("tension_status", np.int32, lambda *d: ()),
    ("tension_iters", np.int32, lambda *d: ()), ("tension_spline", np.float64, lambda P, L, N, R: (9, P)),
    ("tension_length", np.float64, lambda *d: ()),
    ("dp_status", np.int32, lambda *d: ()), ("dp_n_out", np.int32, lambda *d: ()),
    ("dp_layer_s", np.float64, lambda P, L, N, R: (L,)), ("dp_lower", np.float64, lambda P, L, N, R: (L,)),
    ("dp_upper", np.float64, lambda P, L, N, R: (L,)), ("dp_chosen", np.int32, lambda P, L, N, R: (L,)),
    ("dp_vehicle_l", np.float64, lambda *d: ()),
    ("post_offsets", np.float64, lambda P, L, N, R: (L,)), ("post_status", np.int32, lambda *d: ()),
    ("post_iters", np.int32, lambda *d: ()),
    ("ref_spline", np.float64, lambda P, L, N, R: (9, L)), ("max_s", np.float64, lambda *d: ()),
    ("states", np.float64, lambda P, L, N, R: (4, N)), ("curvature", np.float64, lambda P, L, N, R: (N,)),
    ("total", np.int32, lambda *d: ()), ("bounds", np.float64, lambda P, L, N, R: (6, N)),
    ("n_valid", np.int32, lambda *d: ()), ("knots", np.float64, lambda P, L, N, R: (abi.NFIELDS, N)),
    ("inst", np.float64, lambda *d: (abi.NINST,)), ("p", np.int32, lambda *d: ()),
    ("sol1", np.float64, lambda P, L, N, R: (4, N)), ("status1", np.int32, lambda *d: ()),
    ("iters1", np.int32, lambda *d: ()),
    ("x_full1", np.float64, lambda P, L, N, R: (6 * N - 1,)), ("y_full1", np.float64, lambda P, L, N, R: (6 * N + 2,)),
    ("z_full1", np.float64, lambda P, L, N, R: (6 * N + 2,)),
    ("x_full2", np.float64, lambda P, L, N, R: (6 * N - 1,)), ("y_full2", np.float64, lambda P, L, N, R: (6 * N + 2,)),
    ("z_full2", np.float64, lambda P, L, N, R: (6 * N + 2,)),
    ("tension_clearance", np.float64, lambda P, L, N, R: (P,)),
]


class PlanTrace(C.Structure):
    _fields_ = [(n, C.c_void_p) for n, _, _ in _TRACE]


class PlanOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("status", "n", "path", "cost", "iters")] + [("trace", C.POINTER(PlanTrace))]


def _lib():
    L = solver.load_library()
    bounds._declare(L)
    if not getattr(L, "_plan_declared", False):
        vp = C.c_void_p
        L.pqp_plan_default_params.argtypes = [C.POINTER(PlanParams)]
        L.pqp_plan_default_params.restype = None
        L.pqp_plan_create.argtypes = [C.POINTER(bounds.BoundsMap), C.POINTER(PlanParams)] + [C.c_int32] * 6 + [C.POINTER(vp)]
        L.pqp_plan_destroy.argtypes = [vp]
        L.pqp_plan_destroy.restype = None
        L.pqp_plan.argtypes = [vp, C.POINTER(PlanIn), C.POINTER(PlanOut)]
        L.pqp_plan_device.argtypes = [vp, C.POINTER(PlanIn), C.POINTER(PlanOut), vp]
        L.pqp_plan_last_stage_ms.argtypes = [vp, C.POINTER(C.c_float)]
        L.pqp_plan_launch_count.argtypes = [vp, C.POINTER(C.c_int64)]
        L.pqp_plan_last_error.argtypes = [vp]
        L.pqp_plan_last_error.restype = C.c_char_p
        L._plan_declared = True
    return L


def default_params(smoothing_method=None):
    """Library defaults; `smoothing_method` ("TENSION2", "TENSION" or SMOOTH_*) overrides the default TENSION2."""
    p = PlanParams()
    _lib().pqp_plan_default_params(C.byref(p))
    if smoothing_method is not None:
        p.smoothing_method = SMOOTHING_METHODS.get(smoothing_method, smoothing_method)
    return p


class PlanResult:
    """Outputs of one plan call (numpy, host). `trace` is a dict of the stage arrays when requested."""

    def __init__(self, batch, n_max):
        self.status = np.zeros(batch, dtype=np.int32)
        self.n = np.zeros(batch, dtype=np.int32)
        self.path = np.zeros((batch, len(PATH_ROWS), n_max))
        self.cost = np.zeros(batch)
        self.iters = np.zeros((batch, 2), dtype=np.int32)
        self.trace = None

    def status_names(self):
        return [STATUS_NAMES[int(s)] for s in self.status]

    def final_path(self, b):
        """dict of the SlState rows of path b, cut to its n."""
        n = int(self.n[b])
        return {name: self.path[b, i, :n] for i, name in enumerate(PATH_ROWS)}


def _trace_arrays(batch, dims, alloc):
    return {n: alloc((batch,) + shape(*dims), dt) for n, dt, shape in _TRACE}


def _trace_struct(arrays, ptr):
    return PlanTrace(*(ptr(arrays[n]) for n, _, _ in _TRACE))


class Planner:
    """Batched PathOptimizer::solve over one obstacle map (`dist`: float32 distance layer [rows, cols])."""

    def __init__(self, dist, resolution, *, r_max, p_max, layers_max=64, n_max=256, batch_max, center=(0.0, 0.0),
                 params=None, device=0):
        self.L = _lib()
        self.dist = np.ascontiguousarray(dist, dtype=np.float32)
        self.params = params if params is not None else default_params()
        self.r_max, self.p_max, self.layers_max, self.n_max = int(r_max), int(p_max), int(layers_max), int(n_max)
        self.batch_max, self.device = int(batch_max), int(device)
        m = bounds.BoundsMap(self.dist.shape[0], self.dist.shape[1], float(resolution), float(center[0]),
                             float(center[1]), self.dist.ctypes.data)
        h = C.c_void_p()
        rc = self.L.pqp_plan_create(C.byref(m), C.byref(self.params), self.r_max, self.p_max, self.layers_max, self.n_max,
                                    self.batch_max, self.device, C.byref(h))
        if rc:
            raise solver.PqpError(rc, (self.L.pqp_plan_last_error(None) or b"").decode())
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.pqp_plan_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc:
            raise solver.PqpError(rc, (self.L.pqp_plan_last_error(self.h) or b"").decode())

    @property
    def dims(self):
        return self.p_max, self.layers_max, self.n_max, self.r_max

    def plan(self, raw_x, raw_y, start, target, trace=False) -> PlanResult:
        """Host call. raw_x, raw_y: lists of per-path sample arrays (x_list_, y_list_ of bSpline()); start [B][4]
        (x, y, heading, k); target [B][3] (x, y, heading)."""
        B = len(raw_x)
        r = np.array([len(v) for v in raw_x], dtype=np.int32)
        rx, ry = np.zeros((B, self.r_max)), np.zeros((B, self.r_max))
        for b in range(B):
            rx[b, :r[b]], ry[b, :r[b]] = raw_x[b], raw_y[b]
        start = np.ascontiguousarray(start, dtype=np.float64).reshape(B, 4)
        target = np.ascontiguousarray(target, dtype=np.float64).reshape(B, 3)
        res = PlanResult(B, self.n_max)
        pin = PlanIn(B, self.r_max, rx.ctypes.data, ry.ctypes.data, r.ctypes.data, start.ctypes.data, target.ctypes.data)
        tr = None
        if trace:
            res.trace = _trace_arrays(B, self.dims, lambda shape, dt: np.zeros(shape, dtype=dt))
            tr = _trace_struct(res.trace, lambda a: a.ctypes.data)
        pout = PlanOut(res.status.ctypes.data, res.n.ctypes.data, res.path.ctypes.data, res.cost.ctypes.data,
                       res.iters.ctypes.data, C.pointer(tr) if tr is not None else None)
        self._check(self.L.pqp_plan(self.h, C.byref(pin), C.byref(pout)))
        return res

    def plan_device(self, raw_x, raw_y, r, start, target, *, trace=False, stream=None):
        """Device call on torch tensors (cuda, contiguous): raw_x / raw_y float64 [B][r_max'], r int32 [B], start
        float64 [B][4], target float64 [B][3]. Asynchronous on `stream` (default: the current stream); returns a dict of
        output tensors (status, n, path, cost, iters, and `trace`: a dict of tensors when requested)."""
        import torch
        B = int(raw_x.shape[0])
        dev = raw_x.device
        for t in (raw_x, raw_y, r, start, target):
            assert t.is_cuda and t.is_contiguous()
        out = {"status": torch.zeros(B, dtype=torch.int32, device=dev), "n": torch.zeros(B, dtype=torch.int32, device=dev),
               "path": torch.zeros((B, len(PATH_ROWS), self.n_max), dtype=torch.float64, device=dev),
               "cost": torch.zeros(B, dtype=torch.float64, device=dev),
               "iters": torch.zeros((B, 2), dtype=torch.int32, device=dev)}
        tdt = {np.float64: torch.float64, np.int32: torch.int32}
        tr = None
        if trace:
            out["trace"] = _trace_arrays(B, self.dims, lambda shape, dt: torch.zeros(shape, dtype=tdt[dt], device=dev))
            tr = _trace_struct(out["trace"], lambda a: a.data_ptr())
        pin = PlanIn(B, int(raw_x.shape[1]), raw_x.data_ptr(), raw_y.data_ptr(), r.data_ptr(), start.data_ptr(),
                     target.data_ptr())
        pout = PlanOut(out["status"].data_ptr(), out["n"].data_ptr(), out["path"].data_ptr(), out["cost"].data_ptr(),
                       out["iters"].data_ptr(), C.pointer(tr) if tr is not None else None)
        s = stream if stream is not None else torch.cuda.current_stream(dev)
        self._check(self.L.pqp_plan_device(self.h, C.byref(pin), C.byref(pout), C.c_void_p(s.cuda_stream)))
        return out

    @property
    def last_stage_ms(self):
        ms = (C.c_float * len(STAGES))()
        self._check(self.L.pqp_plan_last_stage_ms(self.h, ms))
        return dict(zip(STAGES, (float(v) for v in ms)))

    @property
    def launch_count(self):
        c = C.c_int64(0)
        self._check(self.L.pqp_plan_launch_count(self.h, C.byref(c)))
        return c.value
