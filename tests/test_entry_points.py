"""The host, device and mapped entry points of the map-reading operations agree (GPU): bounds compute, DP search, and
the whole plan from samples and from reference points, each over a handle with three map slots.

Per operation: the host form and the device form (called through ctypes on device buffers) give the same outputs bit
for bit, unmapped and mapped with a mixed index that holds an out-of-range entry; a mapped call with an all-zero index
equals the unmapped call; a mapped call with a NULL index is refused with PQP_E_INVALID and a reason.
"""
import ctypes as C

import numpy as np
import pytest

from path_optimizer_2_b200 import abi, bounds, dp, plan, sharedmap

B = 12
R_MAX, P_MAX, L_MAX, N_MAX = 64, 64, 64, 255
# slots 0 .. 2, and one entry past the last slot
MIXED = np.array([0, 1, 2, 0, 2, 3, 1, 0, 0, 2, 1, 0], np.int32)


@pytest.fixture(scope="module")
def fx():
    """Three maps (the demo map, flipped along each axis), reference lines and plan inputs on the demo map."""
    dmap = sharedmap.DistanceMap()
    layers = [dmap.dist, np.ascontiguousarray(dmap.dist[::-1]), np.ascontiguousarray(dmap.dist[:, ::-1])]
    lines = sharedmap.make_lines(B, 120, dmap=dmap)
    return dict(layers=layers, lines=lines, raw=sharedmap.make_plan_inputs(B, dmap=dmap, lines=lines),
                pts=sharedmap.make_plan_points(B, dmap=dmap))


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _run_device(call):
    """`call`(stream) through ctypes on the current stream, then wait for it."""
    import torch
    rc = call(C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc


def _indices():
    return ((None, "unmapped"), (MIXED, "mixed"))


def _refuses_null_index(rc, last_error, h):
    assert rc == abi.PQP_E_INVALID
    assert b"map_index" in (last_error(h) or b"")


@pytest.mark.gpu
def test_gpu_bounds_compute_entry_points(fx):
    import torch
    ln = fx["lines"]
    pbn = bounds.PathBounds.from_maps(fx["layers"], sharedmap.RES)
    L = pbn.L
    n_max, k_max = ln.states.shape[2], ln.spline.shape[2]
    din = [_cuda(ln.states), _cuda(ln.n), _cuda(ln.spline), _cuda(ln.k)]
    bi = bounds.BoundsIn(B, n_max, k_max, *(t.data_ptr() for t in din))
    for idx, tag in _indices():
        host_b, host_nv = pbn.compute(ln.states, ln.n, ln.spline, ln.k, map_index=idx)
        dev_b = torch.zeros((B, bounds.BOUND_ROWS, n_max), dtype=torch.float64, device="cuda")
        dev_nv = torch.zeros(B, dtype=torch.int32, device="cuda")
        bo = bounds.BoundsOut(dev_b.data_ptr(), dev_nv.data_ptr(), None)
        if idx is None:
            rc = _run_device(lambda s: L.pqp_bounds_compute_device(pbn.h, C.byref(bi), C.byref(bo), s))
        else:
            tidx = _cuda(idx)
            rc = _run_device(lambda s: L.pqp_bounds_compute_mapped_device(pbn.h, C.byref(bi), tidx.data_ptr(),
                                                                         C.byref(bo), s))
        assert rc == 0, tag
        dev_b, dev_nv = dev_b.cpu().numpy(), dev_nv.cpu().numpy()
        assert np.array_equal(host_nv, dev_nv), tag
        for b in range(B):
            assert np.array_equal(host_b[b, :, :host_nv[b]], dev_b[b, :, :dev_nv[b]]), (tag, b)
        if idx is not None:
            assert host_nv[MIXED >= len(fx["layers"])].max() == 0
    zb, znv = pbn.compute(ln.states, ln.n, ln.spline, ln.k, map_index=np.zeros(B, np.int32))
    ub, unv = pbn.compute(ln.states, ln.n, ln.spline, ln.k)
    assert np.array_equal(znv, unv) and unv.min() > 0
    for b in range(B):
        assert np.array_equal(zb[b, :, :unv[b]], ub[b, :, :unv[b]]), b
    # NULL map_index
    host_b, host_nv = np.zeros((B, bounds.BOUND_ROWS, n_max)), np.zeros(B, np.int32)
    hbi = bounds.BoundsIn(B, n_max, k_max, ln.states.ctypes.data, ln.n.ctypes.data, ln.spline.ctypes.data,
                          ln.k.ctypes.data)
    hbo = bounds.BoundsOut(host_b.ctypes.data, host_nv.ctypes.data, None)
    _refuses_null_index(L.pqp_bounds_compute_mapped(pbn.h, C.byref(hbi), None, C.byref(hbo)), L.pqp_bounds_last_error,
                        pbn.h)
    bo = bounds.BoundsOut(dev_b.ctypes.data, dev_nv.ctypes.data, None)
    _refuses_null_index(L.pqp_bounds_compute_mapped_device(pbn.h, C.byref(bi), None, C.byref(bo), None),
                        L.pqp_bounds_last_error, pbn.h)
    pbn.close()


_DP_MAIN = ("status", "n_layers", "n_out", "layer_s", "lower", "upper", "chosen", "vehicle_l", "target_s")


@pytest.mark.gpu
def test_gpu_dp_search_entry_points(fx):
    import torch
    ln = fx["lines"]
    pbn = bounds.PathBounds.from_maps(fx["layers"], sharedmap.RES)
    ds = dp.DpSearch(pbn, layers_max=160, batch_max=B)
    L = ds.L
    length = np.array([ln.spline_rows(b)[0, ln.k[b] - 1] + 3.0 for b in range(B)])
    start = np.ascontiguousarray(np.stack([ln.states[:, 1, 2], ln.states[:, 2, 2], ln.states[:, 3, 2]], axis=1))
    din_t = [_cuda(ln.spline), _cuda(ln.k), _cuda(length), _cuda(start)]
    di = dp.DpIn(B, ln.spline.shape[2], *(t.data_ptr() for t in din_t))
    for idx, tag in _indices():
        host = ds.search(ln.spline, ln.k, length, start, map_index=idx)
        ref = dp.DpResult(B, ds.layers_max, ds.lateral)
        dev = {k: torch.from_numpy(np.zeros_like(getattr(ref, k))).cuda() for k in _DP_MAIN + ("cost", "parent",
                                                                                                "feasible")}
        do = dp.DpOut(*(dev[k].data_ptr() for k in _DP_MAIN + ("cost", "parent", "feasible")))
        if idx is None:
            rc = _run_device(lambda s: L.pqp_dp_search_device(ds.h, C.byref(di), C.byref(do), s))
        else:
            tidx = _cuda(idx)
            rc = _run_device(lambda s: L.pqp_dp_search_mapped_device(ds.h, C.byref(di), tidx.data_ptr(), C.byref(do),
                                                                     s))
        assert rc == 0, tag
        dev = {k: v.cpu().numpy() for k, v in dev.items()}
        for k in _DP_MAIN[:-2]:
            assert np.array_equal(getattr(host, k), dev[k]), (tag, k)
        for b in range(B):
            if host.status[b] != dp.DP_MAP_INDEX:  # a path without a map leaves the vehicle fields unwritten
                for k in _DP_MAIN[-2:]:
                    assert getattr(host, k)[b] == dev[k][b], (tag, b, k)
            nl = int(host.n_layers[b])
            for k in ("cost", "parent", "feasible"):
                assert np.array_equal(getattr(host, k)[b][:nl], dev[k][b][:nl]), (tag, b, k)
        if idx is not None:
            assert (host.status[MIXED >= len(fx["layers"])] == dp.DP_MAP_INDEX).all()
    zero = ds.search(ln.spline, ln.k, length, start, map_index=np.zeros(B, np.int32))
    unmapped = ds.search(ln.spline, ln.k, length, start)
    for k in _DP_MAIN + ("cost", "parent", "feasible"):
        assert np.array_equal(getattr(zero, k), getattr(unmapped, k)), k
    # NULL map_index
    hdi = dp.DpIn(B, ln.spline.shape[2], ln.spline.ctypes.data, ln.k.ctypes.data, length.ctypes.data,
                  start.ctypes.data)
    out = dp.DpResult(B, ds.layers_max, ds.lateral)
    _refuses_null_index(L.pqp_dp_search_mapped(ds.h, C.byref(hdi), None, C.byref(out.as_struct())),
                        L.pqp_dp_last_error, ds.h)
    _refuses_null_index(L.pqp_dp_search_mapped_device(ds.h, C.byref(di), None, C.byref(do), None),
                        L.pqp_dp_last_error, ds.h)
    ds.close()
    pbn.close()


_PLAN_OUT = ("status", "n", "path", "cost", "iters")


def _padded(xs):
    cnt = np.array([len(v) for v in xs], np.int32)
    a = np.zeros((len(xs), R_MAX))
    for b, v in enumerate(xs):
        a[b, :len(v)] = v
    return a, cnt


@pytest.mark.gpu
@pytest.mark.parametrize("points", (False, True), ids=("samples", "points"))
def test_gpu_plan_entry_points(fx, points):
    import torch
    pl = plan.Planner.from_maps(fx["layers"], sharedmap.RES, r_max=R_MAX, p_max=P_MAX, layers_max=L_MAX, n_max=N_MAX,
                                batch_max=B)
    L = pl.L
    xs, ys, start, target = fx["pts" if points else "raw"]
    host_fn = pl.plan_points if points else pl.plan
    make_in = plan.PlanPointsIn if points else plan.PlanIn
    name = "pqp_plan_points" if points else "pqp_plan"
    px, cnt = _padded(xs)
    py, _ = _padded(ys)
    dev_in = [_cuda(px), _cuda(py), _cuda(cnt), _cuda(start), _cuda(target)]
    pin = make_in(B, R_MAX, *(t.data_ptr() for t in dev_in))
    for idx, tag in _indices():
        host = host_fn(xs, ys, start, target, map_index=idx)
        ref = plan.PlanResult(B, N_MAX)
        dev = {k: torch.from_numpy(np.zeros_like(getattr(ref, k))).cuda() for k in _PLAN_OUT}
        pout = plan.PlanOut(*(dev[k].data_ptr() for k in _PLAN_OUT), None)
        if idx is None:
            rc = _run_device(lambda s: getattr(L, name + "_device")(pl.h, C.byref(pin), C.byref(pout), s))
        else:
            tidx = _cuda(idx)
            rc = _run_device(lambda s: getattr(L, name + "_mapped_device")(pl.h, C.byref(pin), tidx.data_ptr(),
                                                                          C.byref(pout), s))
        assert rc == 0, tag
        for k in _PLAN_OUT:
            assert np.array_equal(getattr(host, k), dev[k].cpu().numpy()), (tag, k)
        if idx is None:
            assert (host.status == plan.OK).sum() > B // 2, host.status_names()
        else:
            assert (host.status[MIXED >= len(fx["layers"])] == plan.MAP_INDEX).all()
    zero = host_fn(xs, ys, start, target, map_index=np.zeros(B, np.int32))
    unmapped = host_fn(xs, ys, start, target)
    for k in _PLAN_OUT:
        assert np.array_equal(getattr(zero, k), getattr(unmapped, k)), k
    # NULL map_index
    hx, hy = np.ascontiguousarray(px), np.ascontiguousarray(py)
    hin = make_in(B, R_MAX, hx.ctypes.data, hy.ctypes.data, cnt.ctypes.data, np.ascontiguousarray(start).ctypes.data,
                  np.ascontiguousarray(target).ctypes.data)
    res = plan.PlanResult(B, N_MAX)
    hout = plan.PlanOut(*(getattr(res, k).ctypes.data for k in _PLAN_OUT), None)
    _refuses_null_index(getattr(L, name + "_mapped")(pl.h, C.byref(hin), None, C.byref(hout)), L.pqp_plan_last_error,
                        pl.h)
    _refuses_null_index(getattr(L, name + "_mapped_device")(pl.h, C.byref(pin), None, C.byref(pout), None),
                        L.pqp_plan_last_error, pl.h)
    pl.close()
