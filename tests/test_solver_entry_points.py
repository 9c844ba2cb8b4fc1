"""The path-QP solver's host entry points against its device entry points, bit for bit, on each host pipeline.

`pqp_solve` / `pqp_resolve` stage a batch through the handle's buffers (a streamed persistent launch at B >= 512 on a
persistent handle, a chunked multi-stream pipeline otherwise, one chunk for small batches); `pqp_solve_device` /
`pqp_resolve_device` run the same kernel on the caller's buffers. With the FP64 re-solve off (option bit 4; the device
forms never escalate) every output must agree bit for bit: sol, cost, status, iters, info and x/y/z_full, cold and on
two warm re-solves. The FP64 re-solve of the host forms is checked against an FP64 handle, instance by instance, and
the handle's device-resident results (`pqp_resident_results`, pqp_multi.h) against the host outputs. The layout of a
batch itself is checked on the CPU (tests/cpp/batch_layout_test.cpp under g++)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from path_optimizer_2_b200 import abi, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("sol", "cost", "status", "iters", "info", "x_full", "y_full", "z_full")


def test_batch_layout_table(tmp_path):
    """The per-instance element counts of every pqp_batch_in / pqp_batch_out member, and batch_from's offsets."""
    exe = str(tmp_path / "batch_layout_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
                           "-o", exe, os.path.join(ROOT, "tests", "cpp", "batch_layout_test.cpp")])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok 4 8", out.stdout


# ---------------------------------------------------------------------------------------------------------------- GPU

def _same(a, b):
    a = a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)
    b = b.cpu().numpy() if hasattr(b, "cpu") else np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _assert_same(host, dev, label, idx=None):
    for f in FIELDS:
        h, d = getattr(host, f), getattr(dev, f)
        if idx is not None:
            h, d = h[idx], d[idx]
        assert _same(h, d), "%s: %s differs" % (label, f)


class _DeviceBatch:
    """A HostBatch on the device, full outputs zeroed before every call, and the ABI structs over both."""

    def __init__(self, hb):
        import torch
        dev = torch.device("cuda", 0)
        self.torch, self.dev, self.B, self.n_max = torch, dev, hb.batch, hb.n_max
        self.knots = torch.from_numpy(hb.knots).to(dev)
        self.inst = torch.from_numpy(hb.inst).to(dev)
        self.n = torch.from_numpy(hb.n).to(dev)
        self.p = None if hb.p is None else torch.from_numpy(hb.p).to(dev)
        ref = abi.HostResult(hb.batch, hb.n_max, full=True)
        self.out = {f: torch.from_numpy(getattr(ref, f)).to(dev) for f in FIELDS}

    def set_knots(self, knots):
        self.knots.copy_(self.torch.from_numpy(np.ascontiguousarray(knots)))

    def structs(self):
        for f in ("x_full", "y_full", "z_full"):
            self.out[f].zero_()
        o = self.out
        bi = abi.PqpBatchIn(self.B, self.n_max, self.knots.data_ptr(), self.inst.data_ptr(), self.n.data_ptr(),
                            None if self.p is None else self.p.data_ptr())
        bo = abi.PqpBatchOut(*(o[f].data_ptr() for f in ("sol", "cost", "status", "iters", "x_full", "y_full",
                                                          "z_full", "info")))
        return bi, bo

    def result(self):
        self.torch.cuda.synchronize()
        r = abi.HostResult(self.B, self.n_max, full=True)
        for f in FIELDS:
            setattr(r, f, self.out[f].cpu().numpy())
        return r


# (label, option bits, n, batch, p given): the streamed launch (persistent default at n = 240, B >= 512), the chunked
# pipeline with an uneven last chunk (three chunks of 834, 834, 832), and one chunk with rough constraints (p < n)
CASES = [("streamed", 0, 240, 1024, False), ("chunked", 16, 240, 2500, False), ("single", 0, 120, 7, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("label,bits,n,B,with_p", CASES, ids=[c[0] for c in CASES])
def test_host_form_matches_device_form(label, bits, n, B, with_p):
    from path_optimizer_2_b200 import solver
    params = abi.default_params(reserved=4 | bits)  # no FP64 re-solve: the device forms never escalate
    hb = synthetic.make_batch(7, B, n, ragged=True)
    if with_p:
        hb = abi.HostBatch(hb.knots, hb.inst, hb.n, p=hb.n * np.arange(B) // max(B - 1, 1))
    sh = solver.PathQpSolver(params, n_max=n, batch_max=B)
    sd = solver.PathQpSolver(params, n_max=n, batch_max=B)
    db = _DeviceBatch(hb)
    stream = db.torch.cuda.current_stream().cuda_stream

    res = sh.solve(hb, full=True)
    sd.solve_device(*db.structs(), stream=stream)
    _assert_same(res, db.result(), label + " cold")

    # warm, with new linearisation points from the caller
    hb2 = hb.with_linearisation(res.sol)
    res = sh.resolve(hb2, full=True)
    db.set_knots(hb2.knots)
    sd.solve_device(*db.structs(), stream=stream, warm=True)
    _assert_same(res, db.result(), label + " warm")

    # warm, linearised on the device about the previous solution
    res = sh.resolve(None, batch=B, full=True)
    sd.relinearise_device(B, db.out["sol"].data_ptr(), db.knots.data_ptr(), stream=stream)
    sd.solve_device(*db.structs(), stream=stream, warm=True)
    _assert_same(res, db.result(), label + " warm relinearised")
    sh.close()
    sd.close()


class _DeviceArray:
    """A raw device pointer of the library, readable through torch"""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 2}


def _resident(sv, B, n_max):
    import torch
    from path_optimizer_2_b200 import multi
    L = multi._lib()
    ptrs = [C.c_void_p() for _ in range(4)]
    sv._check(L.pqp_resident_results(sv.h, *(C.byref(p) for p in ptrs)))
    torch.cuda.synchronize()
    shapes = [((B, 4, n_max), "<f8"), ((B,), "<f8"), ((B,), "<i4"), ((B,), "<i4")]
    return [torch.as_tensor(_DeviceArray(p.value, s, t), device="cuda").cpu().numpy() for p, (s, t) in zip(ptrs, shapes)]


@pytest.mark.gpu
@pytest.mark.parametrize("bits,B", [(16, 1300), (8, 700)], ids=["chunked", "streamed"])
def test_escalated_instances_match_an_fp64_handle(bits, B):
    """The suspected-infeasible instances of a host-form solve are re-solved by the FP64 kernel: every output of such
    an instance equals an FP64 handle's; every other instance equals the solve without the re-solve."""
    from path_optimizer_2_b200 import solver
    n = 3
    bad = synthetic.make_batch(103, 6, n)
    hb = synthetic.make_batch(3, B, n)
    at = np.linspace(1, B - 2, 6).astype(int)
    hb.knots[at], hb.inst[at], hb.n[at] = bad.knots, bad.inst, bad.n
    runs = {}
    for name, opt in (("esc", bits), ("fp32", bits | 4), ("fp64", 2)):
        sv = solver.PathQpSolver(abi.default_params(reserved=opt), n_max=n, batch_max=B)
        runs[name] = sv.solve(hb, full=True)
        if name == "esc":
            resident = _resident(sv, B, n)
            stage = sv.last_stage_ms
        sv.close()
    esc, fp32, fp64 = runs["esc"], runs["fp32"], runs["fp64"]
    suspect = np.isin(fp32.status, (abi.PQP_MAX_ITER_REACHED, abi.PQP_PRIMAL_INFEASIBLE_INACCURATE))
    assert suspect[at].any() and abi.PQP_PRIMAL_INFEASIBLE in fp64.status[at]
    if bits == 16:
        assert stage["escalation"] > 0.0
    _assert_same(esc, fp64, "escalated", np.flatnonzero(suspect))
    _assert_same(esc, fp32, "not escalated", np.flatnonzero(~suspect))
    for got, want in zip(resident, (esc.sol, esc.cost, esc.status, esc.iters)):
        assert _same(got, want), "pqp_resident_results against the host outputs"
