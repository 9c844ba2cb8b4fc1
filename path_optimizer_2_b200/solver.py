"""ctypes binding of libpqp_b200.so — the C ABI declared in include/pqp.h.

`PathQpSolver` is the host-side mirror of the reference's `BaseSolver` for a *batch* of
paths: `solve()` is `BaseSolver::solve` (base_solver.cpp:56-95), `resolve()` is
`BaseSolver::updateProblemFormulationAndSolve` (base_solver.cpp:97-117). The object owns
the device buffers and the per-instance warm state the way the reference's solver object
owns its OSQP workspace (base_solver.hpp:62).

There is no CPU path: if the CUDA library is missing or no H100 is visible, construction
raises.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from . import abi

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PQP_LIB_PATH", os.path.join(_PKG, "libpqp_b200.so"))  # override: A/B builds
_CSRC = os.path.join(_PKG, "csrc")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-diag-suppress", "607,177",
              "--shared", "-Xcompiler", "-fPIC"]
_lib = None


class PqpError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("pqp error %d: %s" % (code, msg))
        self.code = code


def build_library(force=False, verbose=False):
    """nvcc-compile the CUDA library in-tree for sm_90a (no GPU needed to compile)."""
    root = os.path.dirname(_PKG)
    cu = [os.path.join(_CSRC, f) for f in ("pqp_api.cu", "pqp_bounds.cu", "pqp_multi.cu", "pqp_smoother.cu")]
    deps = cu + [os.path.join(_CSRC, f) for f in ("pqp_kernel.cuh", "pqp_host_common.h", "pqp_bounds_core.cuh", "pqp_device_guard.h",
                                                  "pqp_dp.cu", "pqp_dp_core.cuh", "pqp_bounds_internal.h", "pqp_smoother_core.cuh",
                                                  "pqp_plan.cu", "pqp_plan_core.cuh", "pqp_smoother_internal.h")]
    deps += [os.path.join(root, "include", f) for f in ("pqp.h", "pqp_bounds.h", "pqp_multi.h", "pqp_dp.h", "pqp_smoother.h",
                                                        "pqp_plan.h")]
    stale = not os.path.exists(LIB_PATH) or any(
        os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in deps)
    if force or stale:
        # the lattice DP (pqp_dp.cu) is a chain of threshold / strict-minimum decisions in FP64, and the plan glue
        # (pqp_plan.cu) is threshold decisions plus spline fits that must equal the host restatement bit for bit: both
        # are compiled without multiply-add contraction so that every operation rounds as in the host restatement
        common = [f for f in NVCC_FLAGS if f != "--shared"] + (["-Xptxas", "-v"] if verbose else []) + [
            "-I", os.path.join(root, "include")]
        objs = []
        for src in ("pqp_dp.cu", "pqp_plan.cu"):
            obj = os.path.join(_PKG, src[:-3] + ".o")
            subprocess.check_call(["nvcc"] + common + ["--fmad=false", "-c", os.path.join(_CSRC, src), "-o", obj])
            objs.append(obj)
        cmd = ["nvcc"] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + [
            "-I", os.path.join(root, "include"), "-o", LIB_PATH] + cu + objs + ["-ldl"]
        subprocess.check_call(cmd)
    return LIB_PATH


def load_library():
    """dlopen the library and declare every symbol of include/pqp.h."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PqpError(abi.PQP_E_NO_DEVICE,
                       "%s not built (run __graft_entry__.build()); there is no CPU fallback" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    pin, pout = C.POINTER(abi.PqpBatchIn), C.POINTER(abi.PqpBatchOut)
    L.pqp_version.restype = C.c_int
    L.pqp_default_params.argtypes = [C.POINTER(abi.PqpParams)]
    L.pqp_create.argtypes = [C.POINTER(abi.PqpParams), C.c_int32, C.c_int32, C.c_int32, C.POINTER(vp)]
    L.pqp_destroy.argtypes = [vp]
    L.pqp_solve.argtypes = [vp, pin, pout]
    L.pqp_resolve.argtypes = [vp, pin, pout]
    L.pqp_solve_device.argtypes = [vp, pin, pout, vp]
    L.pqp_resolve_device.argtypes = [vp, pin, pout, vp]
    L.pqp_relinearise_device.argtypes = [vp, C.c_int32, vp, vp, vp]
    L.pqp_advance_window_device.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, vp, vp, vp, vp, vp]
    L.pqp_frenet_to_cartesian_device.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp]
    L.pqp_frenet_to_cartesian.argtypes = [vp, C.c_int32, vp, vp, vp, vp]
    L.pqp_last_kernel_ms.argtypes = [vp, C.POINTER(C.c_float)]
    L.pqp_launch_count.argtypes = [vp, C.POINTER(C.c_int64)]
    L.pqp_last_stage_ms.argtypes = [vp, C.POINTER(C.c_float)]
    L.pqp_kernel_info.argtypes = [vp, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.pqp_last_error.argtypes = [vp]
    L.pqp_last_error.restype = C.c_char_p
    _lib = L
    return L


EXPORTED_SYMBOLS = [
    "pqp_version", "pqp_default_params", "pqp_create", "pqp_destroy", "pqp_solve", "pqp_resolve",
    "pqp_solve_device", "pqp_resolve_device", "pqp_relinearise_device", "pqp_advance_window_device",
    "pqp_frenet_to_cartesian_device",
    "pqp_frenet_to_cartesian", "pqp_last_kernel_ms", "pqp_last_stage_ms", "pqp_launch_count", "pqp_kernel_info",
    "pqp_last_error",
]


class PathQpSolver:
    """Batched drop-in for the reference's BaseSolver (one handle = batch_max instances)."""

    def __init__(self, params=None, *, n_max, batch_max, device=0):
        self.L = load_library()
        self.params = params if params is not None else abi.default_params()
        self.n_max, self.batch_max, self.device = int(n_max), int(batch_max), int(device)
        h = C.c_void_p()
        rc = self.L.pqp_create(C.byref(self.params), self.n_max, self.batch_max, self.device, C.byref(h))
        if rc:
            raise PqpError(rc, (self.L.pqp_last_error(None) or b"").decode())
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.pqp_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc:
            raise PqpError(rc, (self.L.pqp_last_error(self.h) or b"").decode())

    # ---- host-buffer API (the call a user of the reference makes) -----------------------
    def solve(self, hb: abi.HostBatch, *, full=False, out: abi.HostResult = None) -> abi.HostResult:
        res = out if out is not None else abi.HostResult(hb.batch, hb.n_max, full=full)
        bi, bo = hb.as_struct(), res.as_struct()
        self._check(self.L.pqp_solve(self.h, C.byref(bi), C.byref(bo)))
        return res

    def resolve(self, hb: abi.HostBatch = None, *, full=False, batch=None,
                out: abi.HostResult = None) -> abi.HostResult:
        if hb is None:
            res = out if out is not None else abi.HostResult(batch, self.n_max, full=full)
            bo = res.as_struct()
            self._check(self.L.pqp_resolve(self.h, None, C.byref(bo)))
            return res
        res = out if out is not None else abi.HostResult(hb.batch, hb.n_max, full=full)
        bi, bo = hb.as_struct(), res.as_struct()
        self._check(self.L.pqp_resolve(self.h, C.byref(bi), C.byref(bo)))
        return res

    # ---- device-pointer API (raw addresses, e.g. torch tensors' data_ptr()) --------------
    def solve_device(self, bin_struct: abi.PqpBatchIn, bout_struct: abi.PqpBatchOut, stream=0,
                     warm=False):
        fn = self.L.pqp_resolve_device if warm else self.L.pqp_solve_device
        self._check(fn(self.h, C.byref(bin_struct), C.byref(bout_struct), C.c_void_p(stream)))

    def frenet_to_cartesian(self, n, ref_xyh, sol):
        """getOptimizedPath (base_solver.cpp:263-288) on the device, host buffers."""
        n = np.ascontiguousarray(n, dtype=np.int32)
        ref = np.ascontiguousarray(ref_xyh, dtype=np.float64)
        sol = np.ascontiguousarray(sol, dtype=np.float64)
        out = np.zeros_like(ref)
        self._check(self.L.pqp_frenet_to_cartesian(self.h, len(n), n.ctypes.data, ref.ctypes.data,
                                                   sol.ctypes.data, out.ctypes.data))
        return out

    def relinearise_device(self, batch, sol_ptr, knots_ptr, stream=0):
        """sol -> linearisation fields of the knot block, on the device (pqp_relinearise_device)."""
        self._check(self.L.pqp_relinearise_device(self.h, batch, sol_ptr, knots_ptr, C.c_void_p(stream)))

    def advance_window_device(self, batch, ext_len, tick, ext_ptr, sol_ptr, knots_ptr, inst_ptr, stream=0):
        """Receding-horizon tick bookkeeping on the device (pqp_advance_window_device)."""
        self._check(self.L.pqp_advance_window_device(self.h, batch, ext_len, tick, ext_ptr, sol_ptr, knots_ptr,
                                                     inst_ptr, C.c_void_p(stream)))

    def frenet_to_cartesian_device(self, batch, n_ptr, ref_ptr, sol_ptr, out_ptr, stream=0):
        self._check(self.L.pqp_frenet_to_cartesian_device(self.h, batch, n_ptr, ref_ptr, sol_ptr,
                                                          out_ptr, C.c_void_p(stream)))

    @property
    def last_kernel_ms(self):
        ms = C.c_float(0)
        self._check(self.L.pqp_last_kernel_ms(self.h, C.byref(ms)))
        return ms.value

    STAGES = ("h2d", "kernel", "d2h", "escalation", "total")

    @property
    def last_stage_ms(self):
        """Per-stage device times of the last host-pointer call (pqp_last_stage_ms): the counterpart of
        the TimeRecorder stages of BaseSolver::solve (base_solver.cpp:57-93)."""
        ms = (C.c_float * len(self.STAGES))()
        self._check(self.L.pqp_last_stage_ms(self.h, ms))
        return dict(zip(self.STAGES, (float(v) for v in ms)))

    @property
    def launch_count(self):
        c = C.c_int64(0)
        self._check(self.L.pqp_launch_count(self.h, C.byref(c)))
        return c.value

    @property
    def kernel_info(self):
        a, b, c = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        self._check(self.L.pqp_kernel_info(self.h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(sm_count=a.value, warps_per_sm=b.value, smem_per_warp=c.value)
